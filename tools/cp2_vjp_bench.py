"""Times of the converged 2D TV-L1 backward (proxtv_CP2_TV_* / proxtv_CP2W_TV_* record and vjp, DESIGN.md section 15.2), CUDA events
around device-resident calls after a warmup of every timed call:

  forward   the unrecorded solve (_dev_) and the recorded one (_record_dev_: the same solve, then the fused-edge tape), alg 0, lam 0.2,
            the default 2500 iterations: one 4096 x 4096 float64 image, 8 x 2048 x 2048 float32 images, and the weighted 1024 x 1024
            float64 case (random maps in [0.1, 0.3])
  backward  the vjp on each of those tapes, without and with the weight gradients (glam for the plain solver, gW1 / gW2 for the
            weighted one)
  worst     the backward's worst cases: one cluster over the whole 4096 x 4096 image (lam = 1e9, 20 iterations), and one serpentine
            cluster through a 1024 x 1024 image (zero walls, weights 1e9) that crosses every 32 x 32 tile

Algorithmic bytes of a backward: it reads the upstream gradient and the tape (2 bits per element) and writes gY -- n (2 b + 0.25)
bytes, b the element size -- plus, with weight gradients, X once and each weight map once: n 3 b more.  GB/s is that over the time,
whatever the labelling and the cluster sums actually move.  Prints the card's name, power limit and SM clocks first (read-only
nvidia-smi query) and one JSON line per row.  Changes no device setting.

    python tools/cp2_vjp_bench.py [--steps 3] [--warmup 1] [--out FILE]
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

LAM = 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)

    def emit(r):
        rows.append(r)
        print(json.dumps(r), flush=True)

    def sfx(t):
        return "f32" if t.dtype == torch.float32 else "f64"

    def stream():
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def forward(Y, W, lam, out, info, tape=None, maxit=0):
        B, M, N = Y.shape
        pen = (p(W[0]), p(W[1])) if W else (lam,)
        kind = "CP2W_TV" if W else "CP2_TV"
        if tape is None:
            fn = getattr(lib, "proxtv_%s_dev_%s" % (kind, sfx(Y)))
            ok = fn(M, N, B, 1, p(Y), *pen, p(out), 0, maxit, info.ctypes.data, stream())
        else:
            fn = getattr(lib, "proxtv_%s_record_dev_%s" % (kind, sfx(Y)))
            ok = fn(M, N, B, 1, p(Y), *pen, p(out), 0, maxit, info.ctypes.data, p(tape), tape.numel(), stream())
        assert ok == 1, ptv._lib.last_error()

    def backward(out, tape, g, gY, W, extras):
        B, M, N = out.shape
        if W:
            fn = getattr(lib, "proxtv_CP2W_TV_vjp_dev_%s" % sfx(out))
            ok = fn(M, N, B, 1, p(tape), p(out), p(g), p(gY), *([p(t) for t in extras] if extras else (None, None)), None, stream())
        else:
            fn = getattr(lib, "proxtv_CP2_TV_vjp_dev_%s" % sfx(out))
            ok = fn(M, N, B, 1, p(tape), p(out), p(g), p(gY), p(extras[0]) if extras else None, stream())
        assert ok == 1, ptv._lib.last_error()

    def case(name, Y, W, lam, maxit=0, fwd=True):
        B, M, N = Y.shape
        n, b = B * M * N, Y.element_size()
        out = torch.empty_like(Y); info = np.zeros(3 * B)
        tape = torch.empty(int(lib.proxtv_CP2_TV_tape_bytes(M, N, B)), dtype=torch.uint8, device="cuda")
        if fwd:
            ms0 = timed(lambda: forward(Y, W, lam, out, info, None, maxit), a.steps, a.warmup)
            ms1 = timed(lambda: forward(Y, W, lam, out, info, tape, maxit), a.steps, a.warmup)
            emit({"row": "forward", "case": name, "batch": B, "shape": [M, N], "dtype": sfx(Y), "iters": int(info[0]) - 1,
                  "ms_unrecorded": round(ms0, 2), "ms_recorded": round(ms1, 2)})
        else:
            forward(Y, W, lam, out, info, tape, maxit)
        g = torch.randn_like(Y); gY = torch.empty_like(Y)
        if W:
            extras = (torch.empty_like(W[0]), torch.empty_like(W[1]))
        else:
            extras = (torch.empty(2 * B, dtype=torch.float64, device="cuda"),)
        for with_w in (False, True):
            ms = timed(lambda: backward(out, tape, g, gY, W, extras if with_w else None), a.steps, a.warmup)
            mb = n * (2 * b + 0.25) + (n * 3 * b if with_w else 0)
            emit({"row": "backward", "case": name, "batch": B, "shape": [M, N], "dtype": sfx(Y), "weight_grads": with_w,
                  "ms": round(ms, 3), "model_MB": round(mb / 1e6, 1), "GBps": round(mb / ms / 1e6, 1)})

    case("4096^2 f64", images(1, 4096, 4096, torch.float64), None, LAM)
    case("8x2048^2 f32", images(8, 2048, 2048, torch.float32), None, LAM)
    rng = np.random.default_rng(0)
    M = 1024
    W = (torch.tensor(rng.uniform(0.1, 0.3, (1, M - 1, M)), device="cuda"), torch.tensor(rng.uniform(0.1, 0.3, (1, M, M - 1)), device="cuda"))
    case("weighted 1024^2 f64", images(1, M, M, torch.float64), W, None)
    case("one cluster 4096^2 f64", images(1, 4096, 4096, torch.float64), None, 1e9, maxit=20, fwd=False)
    W1 = np.zeros((1, M - 1, M)); W1[0, 0::2, -1] = 1e9; W1[0, 1::2, 0] = 1e9
    W = (torch.tensor(W1, device="cuda"), torch.full((1, M, M - 1), 1e9, dtype=torch.float64, device="cuda"))
    case("serpentine 1024^2 f64", images(1, M, M, torch.float64), W, None, maxit=20, fwd=False)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
