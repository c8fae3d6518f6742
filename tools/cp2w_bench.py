"""Times of the weighted primal-dual 2D TV-L1 prox (tv1w_2d method 'condat', proxtv_CP2W_TV_dev_*, DESIGN.md section 15.1) against the
weighted Douglas-Rachford splitting (tv1w_2d method 'dr', proxtv_DR2L1W_TV_batched_dev_*), CUDA events around device-resident solves
after a warmup of every timed call:

  solve    condat (alg 0, the default 2500 iterations) and dr (its default 35 iterations) on one 1024 x 1024 and one 4096 x 4096 float64
           image, and on a batch of 8 x 2048 x 2048 float32 images
  accuracy one 1024 x 1024 float64 image: dr at max_iters 35 / 100 / 300 / 1000 and condat at 250 / 500 / 1000 / 2500 iterations, each
           with its time and its max-abs distance to condat-2500 relative to condat-2500's max-abs

Images are tools/dr2_vjp_bench.py's (16 x 16 blocks plus noise); the weights are uniform per edge, in [0.1, 0.3) along columns and
[0.05, 0.25) along rows, so that the two maps differ.  Algorithmic bytes of condat (model_bytes below): the initialisation reads Y and
writes X and both duals; each iteration reads X, Y, U1, U2, W1, W2 and writes X, U1, U2 -- M N B b (4 + 9 iters) bytes, whatever the
kernels actually move.  The weight maps are read in place, so there is no staging traffic.  The rate is model bytes / time, also as a
fraction of the H100 SXM data-sheet HBM3 rate, 3.35 TB/s.  dr gets no byte model (its passes are not a stencil).  Prints the card's
name, power limit and SM clocks first (read-only nvidia-smi query) and one JSON line per row.  Changes no device setting.

    python tools/cp2w_bench.py [--steps 2] [--warmup 1] [--out FILE]
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


def model_bytes(B, M, N, itemsize, iters):
    return B * M * N * itemsize * (4 + 9 * iters)


def weights(B, M, N, dt):
    gen = torch.Generator(device="cuda").manual_seed(1)
    w1 = 0.1 + 0.2 * torch.rand(B, M - 1, N, generator=gen, device="cuda", dtype=dt)
    w2 = 0.05 + 0.2 * torch.rand(B, M, N - 1, generator=gen, device="cuda", dtype=dt)
    return w1, w2


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

    def stream():
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def condat(Y, W1, W2, out, maxit, info):
        B, M, N = Y.shape
        fn = lib.proxtv_CP2W_TV_dev_f32 if Y.dtype == torch.float32 else lib.proxtv_CP2W_TV_dev_f64
        assert fn(M, N, B, 1, p(Y), p(W1), p(W2), p(out), 0, maxit, info.ctypes.data, stream()) == 1, ptv._lib.last_error()

    def dr(Y, W1, W2, out, maxit, info):
        B, M, N = Y.shape
        fn = lib.proxtv_DR2L1W_TV_batched_dev_f32 if Y.dtype == torch.float32 else lib.proxtv_DR2L1W_TV_batched_dev_f64
        fn(M, N, B, 1, p(Y), p(W1), p(W2), p(out), maxit, info.ctypes.data, stream())
        assert info[2] != 3, ptv._lib.last_error()

    for B, M, dt in ((1, 1024, torch.float64), (1, 4096, torch.float64), (8, 2048, torch.float32)):
        Y = images(B, M, M, dt); W1, W2 = weights(B, M, M, dt); out = torch.empty_like(Y); info = np.zeros(3 * B)
        shape = {"batch": B, "shape": [M, M], "dtype": str(dt).split(".")[-1]}
        ms = timed(lambda: condat(Y, W1, W2, out, 0, info), a.steps, a.warmup)
        iters = info[0::3] - 1
        mb = sum(model_bytes(1, M, M, Y.element_size(), int(k)) for k in iters)
        emit(dict(row="solve", method="condat", **shape, iters=int(iters.max()), ms_per_solve=round(ms, 2),
                  model_GB=round(mb / 1e9, 1), model_TBps=round(mb / ms / 1e9, 3), **{"fraction_of_3.35TBps": round(mb / ms / 1e9 / 3.35, 3)}))
        ms = timed(lambda: dr(Y, W1, W2, out, 0, info), a.steps, a.warmup)
        emit(dict(row="solve", method="dr", **shape, iters=int(info[0]), ms_per_solve=round(ms, 2)))
        del Y, W1, W2, out

    Y = images(1, 1024, 1024, torch.float64)[0]
    W1, W2 = (w[0] for w in weights(1, 1024, 1024, torch.float64))
    ref = ptv.tv1w_2d(Y, W1, W2, method="condat", max_iters=2500)
    scale = float(ref.abs().max())
    for method, its in (("dr", (35, 100, 300, 1000)), ("condat", (250, 500, 1000, 2500))):
        for k in its:
            res = {}

            def run():
                res["x"] = ptv.tv1w_2d(Y, W1, W2, method=method, max_iters=k)
            ms = timed(run, a.steps, a.warmup)
            emit({"row": "accuracy", "method": method, "max_iters": k, "ms": round(ms, 2),
                  "max_rel_dist_to_condat2500": float((res["x"] - ref).abs().max()) / scale})
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
