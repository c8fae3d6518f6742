"""The backward passes of the proximal Dykstra solvers PD_TV and PD2_TV on the host (DESIGN.md section 14), shared by test_pd_vjp_cpu.py
and test_gpu_pd_vjp.py:

* ``forward`` -- K iterations of PD_TV (``pd2=False``: pd_device, k_pd_combine) or PD2_TV (``pd2=True``: pd2_device) in the storage type
  with the device's association, K given (no stop test: the device's stop test only picks K, which the tests take from its info[0]),
  every prox pass a chosen 1D solver over the fibers of one axis (pdr_vjp_emu.exact_prox / slope_prox); returns the output and every
  pass output (all of them reach the result);
* ``backward`` -- the unrolled vector-Jacobian product of include/proxtv_b200.h (proxtv_PD*_TV_vjp_dev_*) restated in numpy: per pass
  vjp_emu.restate under that pass's segmentation, the elementwise steps in the storage type with the kernels' association, and the
  penalty gradients summed in float64 over the passes in backward order;
* ``backward_from_tapes`` -- the same restatement driven by decoded (F, U) segmentation tapes instead of pass outputs;
* ``pass_tapes`` / ``device_pass_tapes`` -- the (F, U) tapes of the host passes / of a device tape buffer.
Arrays are column-major flat arrays of n = prod(ns) elements (pdr_vjp_emu.geom).  PD_TV: pass p = j npen + i is term i's pass of
iteration j.  PD2_TV: pass 2j is the first term's pass of iteration j, 2j + 1 the second's; with one term there is one iteration and one
pass.  In both, pass p belongs to term p % npen."""
import numpy as np

import dr2_vjp_emu as D
import pdr_vjp_emu as R
import vjp_emu
from pdr_vjp_emu import geom, surrogate

MAX_ITERS = 35


def penalties(ws, pd2, T):
    """The penalties the passes use: PD_TV's lambdas[i] *= npen in float64 (as run_pd), PD2_TV's as given; rounded to T."""
    return [T(float(w)) for w in ws] if pd2 else R.scaled(ws, T)


def n_passes(pd2, npen, K):
    return (1 if npen == 1 else 2 * K) if pd2 else K * npen


def forward(prox, y, ns, ws, ds, K, pd2):
    """K iterations (PD2_TV with one term: exactly one) of the solver on the flat column-major array y (dims ns) in y's dtype;
    returns (out, passes), out flat like y."""
    T = y.dtype.type
    k = len(ws)
    lam = penalties(ws, pd2, T)
    passes = []
    if not pd2:
        kk = T(k)
        z = [y.copy() for _ in range(k)]
        x = np.zeros_like(y)
        for _ in range(K):
            p = [prox(z[i], *geom(ns, ds[i]), lam[i]) for i in range(k)]
            passes.extend(p)
            x = np.zeros_like(y)
            for i in range(k):
                x = x + p[i] / kk
            for i in range(k):
                z[i] = z[i] + (x - p[i])
        return x, passes
    assert k in (1, 2)
    x, p, q = y.copy(), np.zeros_like(y), np.zeros_like(y)
    for _ in range(1 if k == 1 else K):
        z = prox(x + p, *geom(ns, ds[0]), lam[0])
        passes.append(z)
        p = p + (x - z)
        if k == 2:
            x = prox(z + q, *geom(ns, ds[1]), lam[1])
            passes.append(x)
            q = q + (z - x)
        else:
            x = z.copy()
    return x, passes


def _run(S, G, k, K, pd2):
    """The recurrences of proxtv_b200/csrc/dr2_vjp.cu: pd_vjp_device; S(p, i, h) -> (gx, gw) of pass p (term i) for the upstream h."""
    T = G.dtype.type
    zero = np.zeros_like(G)
    glam = np.zeros(k)

    def vjp(p, i, h):
        sc, gw = S(p, i, h)
        glam[i] += gw.astype(np.float64).sum()
        return sc

    if not pd2:
        kk = T(k)
        a = [zero.copy() for _ in range(k)]
        gk = G / kk
        h = gk - a[0]
        for j in range(K - 1, -1, -1):
            for i in range(k):
                a[i] = a[i] + vjp(j * k + i, i, h)
                if i + 1 < k:
                    h = gk - a[i + 1]
            s = a[0]
            for i in range(1, k):
                s = s + a[i]
            if j > 0:
                gk = s / kk
                h = gk - a[0]
        return s, glam
    gp, gq = zero.copy(), zero.copy()
    h = G - zero
    for j in range((1 if k == 1 else K) - 1, -1, -1):
        if k == 2:
            gq = gq + vjp(2 * j + 1, 1, h)
            h = gq - gp
        gp = gp + vjp(2 * j if k == 2 else 0, 0, h)
        if j > 0:
            h = gp - gq
    return gp, glam


def backward(passes, G, ns, ws, ds, K, pd2):
    """(gY flat like G, glam float64 (npen,)) for the upstream gradient G (flat, storage type) of forward()'s output.  glam: PD_TV's
    are the gradients of the scaled penalties (the caller's ws_i gets npen glam_i), PD2_TV's those of ws itself."""
    k = len(ws)
    lam = penalties(ws, pd2, G.dtype.type)

    def S(p, i, h):
        nf, ln, inc = geom(ns, ds[i])
        X = passes[p].astype(G.dtype)
        gx, gw = vjp_emu.restate(vjp_emu.from_flat(X, nf, ln, inc), vjp_emu.from_flat(h, nf, ln, inc), lam[i])
        return vjp_emu.to_flat(gx, inc), gw
    return _run(S, G, k, K, pd2)


# ---------------------------------------------------------------------------------------------------------------- tapes
def pass_tapes(passes, ns, ws, ds, pd2):
    """(F, U) of every host pass."""
    k = len(ws)
    lam = penalties(ws, pd2, np.float64)
    return [D.tape_bits(X, *geom(ns, ds[p % k]), lam[p % k]) for p, X in enumerate(passes)]


def device_pass_tapes(raw, n, npen, K, pd2):
    """The (F, U) pairs of the passes of K iterations in a device tape buffer (uint8 numpy array, 256-byte header first)."""
    P = n_passes(pd2, npen, K)
    nw = D.tape_words(n)
    words = np.asarray(raw)[256:256 + P * 2 * nw * 4].view(np.uint32).reshape(P, 2, nw)
    return [(words[p, 0], words[p, 1]) for p in range(P)]


def header(raw):
    """(magic, elem, K, npen, nds, cap) of a device tape buffer's header (dr2_vjp.cu: PdrTapeHeader)."""
    raw = np.asarray(raw)
    magic = int(raw[:8].view(np.uint64)[0])
    elem, K, npen, nds = (int(v) for v in raw[8:24].view(np.int32))
    cap = int(raw[24 + 64 + 64:24 + 64 + 64 + 4].view(np.int32)[0])
    return magic, elem, K, npen, nds, cap


def backward_from_tapes(tapes, G, ns, ds, K, pd2):
    """backward() driven by the (F, U) tapes (pass_tapes / device_pass_tapes) instead of the pass outputs."""
    T = G.dtype.type

    def S(p, i, h):
        nf, ln, inc = geom(ns, ds[i])
        Ys, Ws = surrogate(tapes[p][0], tapes[p][1], nf, ln, inc, T)
        gx, gw = vjp_emu.restate(Ys, vjp_emu.from_flat(h, nf, ln, inc), 0.0, W=Ws)
        return vjp_emu.to_flat(gx, inc), gw
    return _run(S, G, len(ds), K, pd2)
