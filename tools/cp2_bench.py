"""Times of the primal-dual 2D TV-L1 solvers (tv1_2d method 'condat' / 'chambolle-pock', proxtv_CP2_TV_dev_*, DESIGN.md section 15),
CUDA events around device-resident solves after a warmup of every timed call:

  solve    one 4096 x 4096 float64 image, alg 0 (Condat) and 1 (Chambolle-Pock), lam = 0.2, the default 2500 iterations; a batch of
           8 x 2048 x 2048 float32 images, alg 0
  accuracy one 1024 x 1024 float64 image, lam = 0.2: 'dr' (DR2_TV) at max_iters 35 / 100 / 300 / 1000 and condat at 250 / 500 /
           1000 / 2500 iterations, each with its time and its max-abs distance to condat-2500 relative to condat-2500's max-abs

Algorithmic bytes (model_bytes below): the initialisation reads Y and writes X and both duals, and each iteration reads X, Y, U1, U2
and writes X, U1, U2 -- M N B b (4 + 7 iters) bytes, whatever the kernels actually move (the tiles' halo reads are L2 hits).  The
roofline fraction is model bytes / time over the H100 SXM data-sheet HBM3 rate, 3.35 TB/s.  Prints the card's name, power limit and
SM clocks first (read-only nvidia-smi query) and one JSON line per row.  Changes no device setting.

    python tools/cp2_bench.py [--steps 2] [--warmup 1] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import proxtv_b200 as ptv  # noqa: E402
from dr2_vjp_bench import gpu_info, images, p, timed  # noqa: E402

HBM_BPS = 3.35e12
LAM = 0.2


def model_bytes(B, M, N, itemsize, iters):
    return B * M * N * itemsize * (4 + 7 * iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)

    def emit(r):
        rows.append(r)
        print(json.dumps(r), flush=True)

    def cp2(Y, out, alg, maxit, info):
        B, M, N = Y.shape
        fn = lib.proxtv_CP2_TV_dev_f32 if Y.dtype == torch.float32 else lib.proxtv_CP2_TV_dev_f64
        ok = fn(M, N, B, 1, p(Y), LAM, p(out), alg, maxit, info.ctypes.data, C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert ok == 1, ptv._lib.last_error()

    for B, M, dt, algs in ((1, 4096, torch.float64, (0, 1)), (8, 2048, torch.float32, (0,))):
        Y = images(B, M, M, dt); out = torch.empty_like(Y); info = np.zeros(3 * B)
        for alg in algs:
            ms = timed(lambda: cp2(Y, out, alg, 0, info), a.steps, a.warmup)
            iters = int(info[0]) - 1
            assert np.all(info[0::3] == info[0])
            mb = model_bytes(B, M, M, Y.element_size(), iters)
            emit({"row": "solve", "alg": alg, "batch": B, "shape": [M, M], "dtype": str(dt).split(".")[-1], "iters": iters,
                  "ms_per_solve": round(ms, 2), "model_GB": round(mb / 1e9, 1), "model_TBps": round(mb / ms / 1e9, 3),
                  "fraction_of_3.35TBps": round(mb / ms / 1e9 / 3.35, 3)})
        del Y, out

    Y = images(1, 1024, 1024, torch.float64)[0]
    ref = ptv.tv1_2d(Y, LAM, method="condat", max_iters=2500)
    scale = float(ref.abs().max())
    for method, its in (("dr", (35, 100, 300, 1000)), ("condat", (250, 500, 1000, 2500))):
        for k in its:
            res = {}

            def run():
                res["x"] = ptv.tv1_2d(Y, LAM, method=method, max_iters=k)
            ms = timed(run, a.steps, a.warmup)
            emit({"row": "accuracy", "method": method, "max_iters": k, "ms": round(ms, 2),
                  "max_rel_dist_to_condat2500": float((res["x"] - ref).abs().max()) / scale})
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
