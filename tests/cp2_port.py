"""ctypes loader of tests/cp2_port.c, the CPU restatement of CondatChambollePock2_TV that the GPU solver (cp2.cu) is checked against
(test infrastructure only).  The source is compiled on first use with the system C compiler, without FMA contraction, into a
temporary directory of this process, so the repository tree is never written.  reference_cp2_tv() calls the unmodified reference
(oracle/_ref/libproxtv_ref.so); only tests/golden/make_cp2_checks.py needs it."""
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
        d = tempfile.mkdtemp(prefix="proxtv_cp2_port_")
        so = os.path.join(d, "libcp2port.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(_HERE, "cp2_port.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(d, ignore_errors=True)          # the loaded library stays mapped
        lib.orc_cp2_tv.argtypes = [C.c_size_t, C.c_size_t, _dp, C.c_double, _dp, C.c_int, C.c_int, _dp]
        lib.orc_cp2_tv.restype = C.c_int
        _lib = lib
    return _lib


def _run(fn, Y, lam, alg, maxit):
    Y = np.require(np.asarray(Y, dtype=np.float64), requirements=["A", "W", "F"])
    out = np.zeros(Y.shape, order="F"); info = np.zeros(3)
    fn(Y.shape[0], Y.shape[1], _p(Y), float(lam), _p(out), int(alg), int(maxit), _p(info))
    return out, info


def cp2_tv(Y, lam, alg=0, maxit=0):
    """CondatChambollePock2_TV restated (alg 0 Condat, 1 Chambolle-Pock, 2 accelerated): (X, info), info[0] = iterations run + 1."""
    return _run(_load().orc_cp2_tv, Y, lam, alg, maxit)


def reference_cp2_tv(Y, lam, alg=0, maxit=0):
    """The same call on the reference's own CondatChambollePock2_TV (oracle/_ref, built by oracle/build_ref.sh)."""
    from oracle import oracle as O
    fn = O.Ref().lib.CondatChambollePock2_TV
    fn.argtypes = [C.c_size_t, C.c_size_t, _dp, C.c_double, _dp, C.c_short, C.c_int, _dp]
    fn.restype = C.c_int
    return _run(fn, Y, lam, alg, maxit)
