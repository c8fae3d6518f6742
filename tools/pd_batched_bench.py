"""Times of the batched proximal Dykstra solvers (tvgen_batched / proxtv_PD*_TV_batched_*, DESIGN.md section 16), CUDA events around
device-resident torch work after a warmup of every timed call:

  row 1   64 x 256^2 float32, 2 terms (PD2_TV)        tvgen_batched vs a Python loop of tvgen over the items
  row 2   8 x 128^3 float32, 3 terms (PD_TV)          the same
          each in three columns: the no-grad forward, the recorded forward (x requires grad) and the backward (sum(y * G))
  row 3   a mixed batch, 64 x 256^2 float32, 2 terms, max_iters 200: half the items smooth (they stop early), half noisy (they run to
          the cap), against an all-noisy batch of the same size; prints every item's K, sum K_b and B max K_b

Prints the card's name, power limit and SM clocks first (read-only nvidia-smi query) and one JSON line per row.  Changes no device
setting.

    python tools/pd_batched_bench.py [--steps 3] [--warmup 1] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import proxtv_b200 as ptv  # noqa: E402
from dr2_vjp_bench import gpu_info, timed  # noqa: E402


def noisy(shape, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=gen, device="cuda", dtype=torch.float32)


def smooth(shape):
    g = torch.meshgrid(*[torch.arange(n, device="cuda", dtype=torch.float32) for n in shape[1:]], indexing="ij")
    v = sum(torch.sin(c / (40.0 + 7 * a)) for a, c in enumerate(g))
    return v.expand(shape).contiguous()


def arms(x, ws, ds, max_iters, steps, warmup):
    """(ms of [batched, loop] for the no-grad forward, the recorded forward and the backward)"""
    ps = [1] * len(ws)
    G = torch.randn_like(x)

    def fwd_b():
        ptv.tvgen_batched(x, ws, ds, ps, max_iters=max_iters)

    def fwd_l():
        for b in range(x.shape[0]):
            ptv.tvgen(x[b], ws, ds, ps, max_iters=max_iters)
    xr = x.clone().requires_grad_(True)

    def rec_b():
        return ptv.tvgen_batched(xr, ws, ds, ps, max_iters=max_iters)

    def rec_l():
        return [ptv.tvgen(xr[b], ws, ds, ps, max_iters=max_iters) for b in range(x.shape[0])]
    yb = rec_b()
    yl = rec_l()

    def bwd_b():
        torch.autograd.grad(yb, xr, G, retain_graph=True)

    def bwd_l():
        torch.autograd.grad(yl, xr, [G[b] for b in range(x.shape[0])], retain_graph=True)
    out = {}
    for name, fb, fl in (("forward", fwd_b, fwd_l), ("recorded", rec_b, rec_l), ("backward", bwd_b, bwd_l)):
        tb, tl = timed(fb, steps, warmup), timed(fl, steps, warmup)
        out[name] = {"batched_ms": round(tb, 3), "loop_ms": round(tl, 3), "speedup": round(tl / tb, 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    for label, shape, ws, ds in (("64x256^2 f32 PD2_TV", (64, 256, 256), [0.3, 0.3], [1, 2]),
                                 ("8x128^3 f32 PD_TV", (8, 128, 128, 128), [0.2, 0.2, 0.2], [1, 2, 3])):
        r = {"row": label, **arms(noisy(shape, 1), ws, ds, 0, a.steps, a.warmup)}
        r["K"] = ptv.tvgen_batched.last_info[:, 0].astype(int).tolist()
        rows.append(r)
        print(json.dumps(r), flush=True)
    shape, ws, ds, cap = (64, 256, 256), [0.3, 0.3], [1, 2], 200
    mixed = noisy(shape, 2)
    mixed[: shape[0] // 2] = smooth((shape[0] // 2,) + shape[1:])
    allnoisy = noisy(shape, 2)
    r = {"row": "mixed 64x256^2 f32 PD2_TV max_iters=200"}
    for name, x in (("mixed", mixed), ("all_noisy", allnoisy)):
        ms = timed(lambda: ptv.tvgen_batched(x, ws, ds, [1, 1], max_iters=cap), a.steps, a.warmup)
        K = ptv.tvgen_batched.last_info[:, 0].astype(int)
        r[name] = {"ms": round(ms, 3), "sum_K": int(K.sum()), "B_maxK": int(len(K) * K.max()), "K": K.tolist()}
    r["time_ratio"] = round(r["mixed"]["ms"] / r["all_noisy"]["ms"], 3)
    r["sum_K_ratio"] = round(r["mixed"]["sum_K"] / r["all_noisy"]["sum_K"], 3)
    rows.append(r)
    print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
