"""Generates tests/golden/cp2_checks.npz from the UNMODIFIED reference's CondatChambollePock2_TV (src/TV2Dopt.cpp:587-760, compiled
into oracle/_ref/libproxtv_ref.so by oracle/build_ref.sh): the 2D TV-L1 prox by Condat's (alg 0), Chambolle-Pock's (alg 1) and the
accelerated Chambolle-Pock (alg 2) primal-dual iteration.

Inputs are not stored: cases() regenerates them from seeds.  Each output is stored as the SHA-256 digest of its float64 bytes
(equal digests <=> identical arrays) together with info[0] (iterations run + 1).  tests/test_cp2_cpu.py pins the CPU port
(tests/cp2_port.c) to these digests; tests/test_gpu_cp2.py then compares the GPU solver with the port bit for bit.

Run from the repository root with the reference built (PROXTV_REFERENCE_SRC=<reference>/src oracle/build_ref.sh):
    python tests/golden/make_cp2_checks.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cp2_port  # noqa: E402
from oracle import oracle as O  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "cp2_checks.npz")

SHAPES = [(2, 2), (2, 7), (7, 2), (33, 47), (64, 64), (128, 96)]
LAMBDAS = [0.0, 0.01, 0.2, 5.0, 1e3]
MAXITS = [1, 7, 0]
ALGS = [0, 1, 2]


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()).digest(), np.uint8)


def image(k, M, N):
    """The seeded input of shape k: piecewise-constant blocks plus noise (gen_cfg2 with 4 x 4 blocks), column-major."""
    return O.gen_cfg2(M, N, seed=100 + k, block=4)


def special_images():
    """(name, Y, lam): a constant and an all-zero image (both stop after one iteration), and a two-level block image at lam = 10
    (runs all 2500 iterations)."""
    blk = np.zeros((24, 20)); blk[:, 10:] = 3.0
    return [("const", np.full((9, 13), 1.5, order="F"), 0.2), ("zero", np.zeros((9, 13), order="F"), 0.2),
            ("block", np.asfortranarray(blk), 10.0)]


def cases():
    """Every case as (key, Y, lam, alg, maxit), in a fixed order."""
    for k, (M, N) in enumerate(SHAPES):
        Y = image(k, M, N)
        for alg in ALGS:
            for li, lam in enumerate(LAMBDAS):
                for maxit in MAXITS:
                    yield "s%d_a%d_l%d_m%d" % (k, alg, li, maxit), Y, lam, alg, maxit
    for name, Y, lam in special_images():
        for alg in ALGS:
            yield "%s_a%d" % (name, alg), Y, lam, alg, 0


def main():
    out = {}
    for key, Y, lam, alg, maxit in cases():
        X, info = cp2_port.reference_cp2_tv(Y, lam, alg, maxit)
        out[key + "_digest"] = digest(X)
        out[key + "_iters"] = np.array(info[0])
    np.savez_compressed(PATH, **out)
    print("wrote %s (%d cases)" % (PATH, len(out) // 2))


if __name__ == "__main__":
    main()
