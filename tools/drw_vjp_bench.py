"""Times of the DR2L1W_TV backward pass (DESIGN.md section 12) against the no-grad solve (CUDA events, warmup, device-resident buffers):

  4k-f64   one 4096 x 4096 float64 image, column-major, per-edge weights uniform in [0.05, 0.5], 35 iterations
  4k-f32   the same in float32

For each: the no-grad solve (proxtv_DR2L1W_TV_dev_*), the recorded forward (proxtv_DR2L1W_TV_record_dev_*), the backward without and
with both weight gradients (proxtv_DR2L1W_TV_vjp_dev_*), and the tape's size.  Prints one JSON line per shape and the card's name,
power limit and SM clock before and after (read-only nvidia-smi query).  Changes no device setting.

    python tools/drw_vjp_bench.py [--steps 10] [--warmup 2] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    M = N = 4096
    for name, dt in (("4k-f64", torch.float64), ("4k-f32", torch.float32)):
        f32 = dt == torch.float32
        Y = images(1, M, N, dt)[0]                       # read as the column-major buffer of an M x N image
        gen = torch.Generator(device="cuda").manual_seed(1)
        W1 = (0.05 + 0.45 * torch.rand(N, M - 1, generator=gen, device="cuda", dtype=torch.float64)).to(dt)
        W2 = (0.05 + 0.45 * torch.rand(N - 1, M, generator=gen, device="cuda", dtype=torch.float64)).to(dt)
        out = torch.empty_like(Y)
        G = torch.randn_like(Y)
        gY = torch.empty_like(Y)
        gW1, gW2 = torch.empty_like(W1), torch.empty_like(W2)
        nb = lib.proxtv_DR2L1W_TV_tape_bytes(M, N, 0)
        tape = torch.empty(nb, dtype=torch.uint8, device="cuda")
        info = np.zeros(3)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        solve = lib.proxtv_DR2L1W_TV_dev_f32 if f32 else lib.proxtv_DR2L1W_TV_dev_f64
        rec = lib.proxtv_DR2L1W_TV_record_dev_f32 if f32 else lib.proxtv_DR2L1W_TV_record_dev_f64
        vjp = lib.proxtv_DR2L1W_TV_vjp_dev_f32 if f32 else lib.proxtv_DR2L1W_TV_vjp_dev_f64
        ip = C.c_void_p(info.ctypes.data)
        ms_solve = timed(lambda: solve(M, N, p(Y), p(W1), p(W2), p(out), 0, ip, st), a.steps, a.warmup)
        ref = out.clone()
        ms_rec = timed(lambda: rec(M, N, p(Y), p(W1), p(W2), p(out), 0, p(tape), nb, ip, st), a.steps, a.warmup)
        same = bool(torch.equal(out, ref))
        ms_b = timed(lambda: vjp(M, N, 0, p(tape), p(G), p(gY), None, None, st), a.steps, a.warmup)
        ms_bw = timed(lambda: vjp(M, N, 0, p(tape), p(G), p(gY), p(gW1), p(gW2), st), a.steps, a.warmup)
        r = {"shape": name, "M": M, "N": N, "dtype": str(dt).replace("torch.", ""), "solve_ms": round(ms_solve, 3),
             "record_ms": round(ms_rec, 3), "backward_ms": round(ms_b, 3), "backward_gw_ms": round(ms_bw, 3),
             "tape_MiB": round(nb / 2 ** 20, 1), "record_equals_solve": same}
        rows.append(r)
        print(json.dumps(r), flush=True)
        del Y, W1, W2, out, ref, G, gY, gW1, gW2, tape
        torch.cuda.empty_cache()
        lib.proxtv_release_workspace()
    rows.append({"gpu_after": gpu_info()})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
