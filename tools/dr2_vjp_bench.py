"""Times of the DR2_TV backward pass (DESIGN.md section 11) against the no-grad solve (CUDA events, warmup, device-resident buffers):

  4k      one 4096 x 4096 float64 image, row-major, lambda = 0.2, 35 iterations       (BASELINE config 2's shape)
  b16     16 images of 1024 x 1024 float32, row-major, lambda = 0.2, 35 iterations

For each: the no-grad solve (proxtv_DR2_TV_dev_*), the recorded forward (proxtv_DR2_TV_record_dev_*), the backward without and with
the penalty gradients (proxtv_DR2_TV_vjp_dev_*), and the tape's size.  Prints one JSON line per shape and the card's name, power limit
and SM clock before and after (read-only nvidia-smi query).  Changes no device setting.

    python tools/dr2_vjp_bench.py [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import proxtv_b200 as ptv  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable: %s" % e


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def images(B, M, N, dt):
    """Blocks of 16 x 16 plus noise (the BASELINE generator's kind of image)."""
    gen = torch.Generator(device="cuda").manual_seed(0)
    lv = torch.randn(B, M // 16, N // 16, generator=gen, device="cuda", dtype=dt)
    return (lv.repeat_interleave(16, dim=1).repeat_interleave(16, dim=2)
            + 0.3 * torch.randn(B, M, N, generator=gen, device="cuda", dtype=dt)).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    for name, B, M, N, dt in (("4k", 1, 4096, 4096, torch.float64), ("b16", 16, 1024, 1024, torch.float32)):
        f32 = dt == torch.float32
        Y = images(B, M, N, dt)
        out = torch.empty_like(Y)
        G = torch.randn_like(Y)
        gY = torch.empty_like(Y)
        glam = torch.empty(2 * B, dtype=torch.float64, device="cuda")
        nb = lib.proxtv_DR2_TV_tape_bytes(M, N, B, 0)
        tape = torch.empty(nb, dtype=torch.uint8, device="cuda")
        info = np.zeros(3)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        solve = lib.proxtv_DR2_TV_dev_f32 if f32 else lib.proxtv_DR2_TV_dev_f64
        rec = lib.proxtv_DR2_TV_record_dev_f32 if f32 else lib.proxtv_DR2_TV_record_dev_f64
        vjp = lib.proxtv_DR2_TV_vjp_dev_f32 if f32 else lib.proxtv_DR2_TV_vjp_dev_f64
        ip = C.c_void_p(info.ctypes.data)
        ms_solve = timed(lambda: solve(M, N, B, 1, p(Y), 0.2, 0.2, p(out), 0, ip, st), a.steps, a.warmup)
        engine = "lane" if lib.proxtv_lane_guard_last() == 1 else "chunked"
        ms_rec = timed(lambda: rec(M, N, B, 1, p(Y), 0.2, 0.2, p(out), 0, p(tape), nb, ip, st), a.steps, a.warmup)
        ms_b = timed(lambda: vjp(M, N, B, 1, 0, p(tape), p(G), p(gY), None, st), a.steps, a.warmup)
        ms_bl = timed(lambda: vjp(M, N, B, 1, 0, p(tape), p(G), p(gY), p(glam), st), a.steps, a.warmup)
        r = {"shape": name, "B": B, "M": M, "N": N, "dtype": str(dt).replace("torch.", ""), "engine": engine,
             "solve_ms": round(ms_solve, 3), "record_ms": round(ms_rec, 3), "backward_ms": round(ms_b, 3),
             "backward_glam_ms": round(ms_bl, 3), "tape_MiB": round(nb / 2 ** 20, 1)}
        rows.append(r)
        print(json.dumps(r), flush=True)
        del Y, out, G, gY, glam, tape
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
