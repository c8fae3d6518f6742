"""Times of the batched weighted 2D prox (tv1w_2d_batched / proxtv_DR2L1W_TV_batched_*, DESIGN.md section 12), CUDA events around
device-resident work after a warmup of every timed call:

  shapes   64 x 256^2, 16 x 1024^2, 4 x 2048^2 images, float32 and float64, 35 iterations, per-edge weights uniform in [0.05, 0.5]
  arm a    tv1w_2d_batched on the C-ordered batch  vs  a Python loop of tv1w_2d over the same images (torch tensors, no grad)
  arm b    proxtv_DR2L1W_TV_batched_dev_* on the C-ordered batch (row_major = 1)  vs  the per-image column-major batch (row_major = 0)
  arm c    the no-grad solve, the recorded forward (proxtv_DR2L1W_TV_batched_record_dev_*) and the backward with both weight gradients
           (proxtv_DR2L1W_TV_batched_vjp_dev_*), C order

Algorithmic bytes (model_bytes below): per Douglas-Rachford iteration the column pass reads t and W1 and writes s, the row pass reads
Y, s, t and W2 and writes t' -- 8 arrays of the batch's size, K + 1 = 36 times -- whatever the kernels actually move (the strided
pass's gather and scatter add two more sweeps).  GB/s = model bytes / time.  Prints the card's name, power limit and SM clocks first
(read-only nvidia-smi query) and one JSON line per shape.  Changes no device setting.

    python tools/drw_batched_bench.py [--steps 3] [--warmup 1] [--out FILE]
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

SHAPES = ((64, 256, 256), (16, 1024, 1024), (4, 2048, 2048))
K = 35


def model_bytes(B, M, N, itemsize):
    return (K + 1) * 8 * B * M * N * itemsize


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for dt in (torch.float32, torch.float64):
        sfx = "f32" if dt == torch.float32 else "f64"
        solve = getattr(lib, "proxtv_DR2L1W_TV_batched_dev_" + sfx)
        rec = getattr(lib, "proxtv_DR2L1W_TV_batched_record_dev_" + sfx)
        vjp = getattr(lib, "proxtv_DR2L1W_TV_batched_vjp_dev_" + sfx)
        for B, M, N in SHAPES:
            gen = torch.Generator(device="cuda").manual_seed(1)
            Y = images(B, M, N, dt)
            W1 = (0.05 + 0.45 * torch.rand(B, M - 1, N, generator=gen, device="cuda", dtype=torch.float64)).to(dt)
            W2 = (0.05 + 0.45 * torch.rand(B, M, N - 1, generator=gen, device="cuda", dtype=torch.float64)).to(dt)
            info = np.zeros(3)
            ip = C.c_void_p(info.ctypes.data)
            out = torch.empty_like(Y)
            # arm a: the Python surface, batched vs a loop of single-image calls
            with torch.no_grad():
                ms_api = timed(lambda: ptv.tv1w_2d_batched(Y, W1, W2), a.steps, a.warmup)
                ms_loop = timed(lambda: [ptv.tv1w_2d(Y[b], W1[b], W2[b]) for b in range(B)], a.steps, a.warmup)
                same = all(bool(torch.equal(ptv.tv1w_2d_batched(Y, W1, W2)[b], ptv.tv1w_2d(Y[b], W1[b], W2[b]))) for b in (0, B - 1))
            # arm b: storage orders on device buffers
            Yc = Y.transpose(1, 2).contiguous()
            W1c, W2c = W1.transpose(1, 2).contiguous(), W2.transpose(1, 2).contiguous()
            ms_c = timed(lambda: solve(M, N, B, 1, p(Y), p(W1), p(W2), p(out), 0, ip, st), a.steps, a.warmup)
            ref = out.clone()
            outc = torch.empty_like(Yc)
            ms_f = timed(lambda: solve(M, N, B, 0, p(Yc), p(W1c), p(W2c), p(outc), 0, ip, st), a.steps, a.warmup)
            orders_equal = bool(torch.equal(outc.transpose(1, 2), ref))
            del Yc, W1c, W2c, outc
            # arm c: recorded forward and backward
            nb = lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, B, 0)
            tape = torch.empty(nb, dtype=torch.uint8, device="cuda")
            ms_rec = timed(lambda: rec(M, N, B, 1, p(Y), p(W1), p(W2), p(out), 0, p(tape), nb, ip, st), a.steps, a.warmup)
            rec_same = bool(torch.equal(out, ref))
            G, gY = torch.randn_like(Y), torch.empty_like(Y)
            gW1, gW2 = torch.empty_like(W1), torch.empty_like(W2)
            ms_bwd = timed(lambda: vjp(M, N, B, 1, 0, p(tape), p(G), p(gY), p(gW1), p(gW2), st), a.steps, a.warmup)
            del tape, G, gY, gW1, gW2
            mb = model_bytes(B, M, N, Y.element_size())
            row = {"shape": "%dx%dx%d" % (B, M, N), "dtype": sfx,
                   "a_batched_ms": round(ms_api, 3), "a_loop_ms": round(ms_loop, 3), "a_loop_over_batched": round(ms_loop / ms_api, 3),
                   "a_equal": same,
                   "b_corder_ms": round(ms_c, 3), "b_colmajor_ms": round(ms_f, 3), "b_orders_equal": orders_equal,
                   "c_solve_ms": round(ms_c, 3), "c_record_ms": round(ms_rec, 3), "c_backward_ms": round(ms_bwd, 3),
                   "c_record_equal": rec_same, "tape_mib": round(nb / 2 ** 20, 1),
                   "model_gbs_corder": round(mb / (ms_c * 1e6), 1), "model_gbs_colmajor": round(mb / (ms_f * 1e6), 1)}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del Y, W1, W2, out, ref
            torch.cuda.empty_cache()
    rows.append({"gpu_after": gpu_info()})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
