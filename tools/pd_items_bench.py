"""Times of per-item penalties in tvgen_batched (DESIGN.md section 16.1), CUDA events around device-resident torch work after a warmup
of every timed call:

  row 1   64 x 256^2 float32, 2 terms (PD2_TV)
  row 2   8 x 128^3 float32, 3 terms (PD_TV)
          noisy inputs; four arms:
            shared     one ws for every item (the _batched_ call)
            equal      a (B, npen) ws whose rows are all the shared one (the _batched_items_ call; the shared call's kernels)
            distinct   a (B, npen) ws with rows drawn from [0.1, 0.5] (the per-fiber kernels)
            loop       a Python loop of tvgen(x[b], ws[b]) over the distinct rows
          each in three columns: the no-grad forward, the recorded forward (x requires grad) and the backward (sum(y * G)).
          The arms need not run the same iterations: with the shared penalties every item runs the 35-iteration cap, with distinct
          rows some items stop earlier on their own test.  So every column is also given per item-iteration (time / sum_b K_b, in
          microseconds), the like-for-like figure; sum_K is printed with each arm.

Prints the card's name, power limit and SM clocks first (read-only nvidia-smi query) and one JSON line per row.  Changes no device
setting.

    python tools/pd_items_bench.py [--steps 3] [--warmup 1] [--out FILE]
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
from pd_batched_bench import noisy  # noqa: E402


def arm(x, ws, ds, steps, warmup, loop=False):
    """ms of the no-grad forward, the recorded forward and the backward; the K of every item"""
    ps = [1] * len(ds)
    G = torch.randn_like(x)
    xr = x.clone().requires_grad_(True)
    if loop:
        def call(a):
            return [ptv.tvgen(a[b], ws[b], ds, ps) for b in range(x.shape[0])]
    else:
        def call(a):
            return ptv.tvgen_batched(a, ws, ds, ps)
    if loop:
        K = []
        for b in range(x.shape[0]):
            ptv.tvgen(x[b], ws[b], ds, ps)
            K.append(int(ptv.tvgen.last_info[0]))
    else:
        call(x)
        K = ptv.tvgen_batched.last_info[:, 0].astype(int).tolist()
    y = call(xr)

    def bwd():
        if loop:
            torch.autograd.grad(y, xr, [G[b] for b in range(x.shape[0])], retain_graph=True)
        else:
            torch.autograd.grad(y, xr, G, retain_graph=True)
    r = {"forward_ms": round(timed(lambda: call(x), steps, warmup), 3),
         "recorded_ms": round(timed(lambda: call(xr), steps, warmup), 3),
         "backward_ms": round(timed(bwd, steps, warmup), 3), "sum_K": int(sum(K)), "K_range": [min(K), max(K)]}
    for col in ("forward", "recorded", "backward"):
        r[col + "_us_per_item_iter"] = round(1e3 * r[col + "_ms"] / sum(K), 3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    for label, shape, w, ds in (("64x256^2 f32 PD2_TV", (64, 256, 256), [0.3, 0.3], [1, 2]),
                                ("8x128^3 f32 PD_TV", (8, 128, 128, 128), [0.2, 0.2, 0.2], [1, 2, 3])):
        x = noisy(shape, 1)
        B = shape[0]
        distinct = np.random.default_rng(7).uniform(0.1, 0.5, size=(B, len(ds)))
        r = {"row": label}
        for name, ws, loop in (("shared", w, False), ("equal", np.tile(np.array(w), (B, 1)), False), ("distinct", distinct, False),
                               ("loop", distinct, True)):
            r[name] = arm(x, ws, ds, a.steps, a.warmup, loop)
        for col in ("forward", "recorded", "backward"):
            per = col + "_us_per_item_iter"
            r["distinct_over_shared_per_item_iter_" + col] = round(r["distinct"][per] / r["shared"][per], 3)
            r["loop_over_distinct_" + col] = round(r["loop"][col + "_ms"] / r["distinct"][col + "_ms"], 2)
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
