"""ctypes loader of tests/cp2w_port.c, the CPU restatement of the weighted Condat / Chambolle-Pock 2D TV-L1 prox that the GPU solver
(proxtv_CP2W_TV_*, cp2.cu) is checked against (test infrastructure only).  Compiled on first use like tests/cp2_port.py: the system C
compiler, no FMA contraction, a temporary directory of this process, so the repository tree is never written."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_dp = C.POINTER(C.c_double)
_lib = None


def _p(a):
    return a.ctypes.data_as(_dp)


def _load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="proxtv_cp2w_port_")
        so = os.path.join(d, "libcp2wport.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(_HERE, "cp2w_port.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(d, ignore_errors=True)          # the loaded library stays mapped
        lib.orc_cp2w_tv.argtypes = [C.c_size_t, C.c_size_t, _dp, _dp, _dp, _dp, C.c_int, C.c_int, _dp]
        lib.orc_cp2w_tv.restype = C.c_int
        _lib = lib
    return _lib


def _f(a):
    return np.require(np.asarray(a, dtype=np.float64), requirements=["A", "W", "F"])


def cp2w_tv(Y, W1, W2, alg=0, maxit=0):
    """The weighted iteration (alg 0 Condat, 1 Chambolle-Pock) on Y (M, N) with W1 (M-1, N) the weights of the edges along columns
    and W2 (M, N-1) along rows: (X, info), X Fortran-ordered, info[0] = iterations run + 1."""
    Y = _f(Y)
    M, N = Y.shape
    W1 = _f(W1); W2 = _f(W2)
    assert W1.shape == (M - 1, N) and W2.shape == (M, N - 1)
    w1 = np.append(W1.ravel("F"), 0.0); w2 = np.append(W2.ravel("F"), 0.0)       # never empty
    out = np.zeros(Y.shape, order="F"); info = np.zeros(3)
    ok = _load().orc_cp2w_tv(M, N, _p(Y), _p(w1), _p(w2), _p(out), int(alg), int(maxit), _p(info))
    assert ok == 1
    return out, info
