"""A float64 host restatement of the converged 2D TV-L1 backward (proxtv_CP2_TV_vjp_dev_* / proxtv_CP2W_TV_vjp_dev_*, DESIGN.md section
15.2), driven by tests/cp2_dual_port.c, the weighted primal-dual iteration that also returns its final duals (test infrastructure
only).  The C source is compiled on first use like tests/cp2_port.py: the system C compiler, no FMA contraction, a temporary
directory of this process, so the repository tree is never written.

All arrays are (M, N) images in index terms; W1 / U1 / f1 / gw1: (M-1, N), the edges (i, j)-(i+1, j) (axis 0); W2 / U2 / f2 / gw2:
(M, N-1), the edges (i, j)-(i, j+1) (axis 1)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_dp = C.POINTER(C.c_double)
_lib = None


def _load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="proxtv_cp2_dual_port_")
        so = os.path.join(d, "libcp2dualport.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(_HERE, "cp2_dual_port.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(d, ignore_errors=True)          # the loaded library stays mapped
        lib.orc_cp2w_duals.argtypes = [C.c_size_t, C.c_size_t, _dp, _dp, _dp, _dp, _dp, _dp, C.c_int, C.c_int, _dp]
        lib.orc_cp2w_duals.restype = C.c_int
        _lib = lib
    return _lib


def _f(a):
    return np.require(np.asarray(a, dtype=np.float64), requirements=["A", "W", "F"])


def weights(M, N, lam):
    """The maps of the plain solver: every weight lam."""
    return np.full((M - 1, N), float(lam)), np.full((M, N - 1), float(lam))


def solve(Y, W1, W2, alg=0, maxit=0):
    """(X, U1, U2, info) of the weighted iteration (alg 0 / 1); W1 = W2 = lam everywhere is the plain solver bit for bit."""
    Y = _f(Y)
    M, N = Y.shape
    W1, W2 = _f(W1), _f(W2)
    assert W1.shape == (M - 1, N) and W2.shape == (M, N - 1)
    w1 = np.append(W1.ravel("F"), 0.0); w2 = np.append(W2.ravel("F"), 0.0)
    X = np.zeros((M, N), order="F")
    u1 = np.zeros((M - 1) * N + 1); u2 = np.zeros(M * (N - 1) + 1); info = np.zeros(3)
    p = lambda a: a.ctypes.data_as(_dp)  # noqa: E731
    assert _load().orc_cp2w_duals(M, N, p(Y), p(w1), p(w2), p(X), p(u1), p(u2), int(alg), int(maxit), p(info)) == 1
    U1 = u1[:-1].reshape((M - 1, N), order="F"); U2 = u2[:-1].reshape((M, N - 1), order="F")
    return X, U1, U2, info


def fused(X, U1, U2, W1, W2):
    """The fusion rule: w > 0 and (|U| < w or the two values equal); NaN never fuses."""
    with np.errstate(invalid="ignore"):
        f1 = (W1 > 0) & ((np.abs(U1) < W1) | (X[1:, :] == X[:-1, :]))
        f2 = (W2 > 0) & ((np.abs(U2) < W2) | (X[:, 1:] == X[:, :-1]))
    return f1, f2


def labels(f1, f2):
    """Cluster label of every pixel (M, N) from the fused edges: the connected components of the 4-connected fused graph."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    M, N = f1.shape[0] + 1, f2.shape[1] + 1
    idx = np.arange(M * N).reshape((M, N), order="F")
    a = np.concatenate([idx[:-1, :][f1], idx[:, :-1][f2]])
    b = np.concatenate([idx[1:, :][f1], idx[:, 1:][f2]])
    G = coo_matrix((np.ones(a.size), (a, b)), shape=(M * N, M * N))
    return connected_components(G, directed=False)[1].reshape((M, N), order="F")


def vjp(X, f1, f2, g):
    """(gx, gw1, gw2, glam) for the upstream gradient g, in float64: cluster means, the cut edges' sgn(y_j - y_i)(gx_i - gx_j), 0 on
    fused edges, glam = [sum gw1, sum gw2]."""
    lab = labels(f1, f2)
    g = np.asarray(g, dtype=np.float64)
    S = np.bincount(lab.ravel(), weights=g.ravel()); cnt = np.bincount(lab.ravel())
    gx = (S / cnt)[lab]
    gw1 = np.where(f1, 0.0, np.sign(X[1:, :] - X[:-1, :]) * (gx[:-1, :] - gx[1:, :]))
    gw2 = np.where(f2, 0.0, np.sign(X[:, 1:] - X[:, :-1]) * (gx[:, :-1] - gx[:, 1:]))
    return gx, gw1, gw2, np.array([gw1.sum(), gw2.sum()])


def cluster_abs_mean(f1, f2, g):
    """(sum over C of |g|) / |C| per pixel: the scale of the backward's bound."""
    lab = labels(f1, f2)
    S = np.bincount(lab.ravel(), weights=np.abs(np.asarray(g, dtype=np.float64)).ravel()); cnt = np.bincount(lab.ravel())
    return (S / cnt)[lab]
