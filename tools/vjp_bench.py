"""Forward and backward times of the batched 1D prox on three shapes (CUDA events, warmup, device-resident torch buffers):

  cfg3   65536 x 4096 float64, per-edge weights, backward with gw       (BASELINE config 3)
  cfg1   one fiber of 10^6 float64 samples, lam = 0.5                   (BASELINE config 1's shape)
  b4k    4096 fibers x 4096 samples float32, lam = 0.2

The backward's algorithmic bytes are what it must stream: y, g (+ weights) in, gx (+ gw) out; GB/s is reported against the H100 SXM
data sheet's 3350 GB/s.  --sweep also times the backward at forced chunk lengths (proxtv_vjp_tuning).  Prints one JSON line per
measurement and the card's name, power limit and SM clock (read-only nvidia-smi query).  Changes no device setting.

    python tools/vjp_bench.py [--steps 20] [--warmup 3] [--sweep] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import proxtv_b200 as ptv  # noqa: E402

PEAK_GBS = 3350.0


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        return q
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


def make(name):
    gen = torch.Generator(device="cuda").manual_seed(0)
    if name == "cfg3":
        B, L, dt, lam = 65536, 4096, torch.float64, 0.0
        lv = torch.randn(B, L // 64, generator=gen, device="cuda", dtype=dt) * 2
        x = lv.repeat_interleave(64, dim=1) + 0.5 * torch.randn(B, L, generator=gen, device="cuda", dtype=dt)
        w = 0.1 + 0.9 * torch.rand(B, L - 1, generator=gen, device="cuda", dtype=dt)
    elif name == "cfg1":
        B, L, dt, lam = 1, 1_000_000, torch.float64, 0.5
        lv = torch.randn(1, L // 1000, generator=gen, device="cuda", dtype=dt) * 2
        x = lv.repeat_interleave(1000, dim=1) + 0.5 * torch.randn(B, L, generator=gen, device="cuda", dtype=dt)
        w = None
    else:
        B, L, dt, lam = 4096, 4096, torch.float32, 0.2
        lv = torch.randn(B, L // 16, generator=gen, device="cuda", dtype=dt)
        x = lv.repeat_interleave(16, dim=1) + 0.3 * torch.randn(B, L, generator=gen, device="cuda", dtype=dt)
        w = None
    g = torch.randn(B, L, generator=gen, device="cuda", dtype=dt)
    return B, L, lam, x.contiguous(), w, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    info = gpu_info()
    rows = [{"gpu": info}]
    print(json.dumps(rows[0]), flush=True)
    for name in ("cfg3", "cfg1", "b4k"):
        B, L, lam, x, w, g = make(name)
        f32 = x.dtype == torch.float32
        fwd = lib.proxtv_prox_fibers_dev_f32 if f32 else lib.proxtv_prox_fibers_dev_f64
        bwd = lib.proxtv_prox_fibers_vjp_dev_f32 if f32 else lib.proxtv_prox_fibers_vjp_dev_f64
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        y = torch.empty_like(x)
        gx = torch.empty_like(x)
        gw = torch.empty(B, L - 1, dtype=x.dtype, device="cuda")
        ms_f = timed(lambda: fwd(p(x), p(y), B, L, 1, lam, p(w), st), a.steps, a.warmup)
        b = x.element_size()
        n, ne = B * L, B * (L - 1)
        for want_gw in ((True,) if name == "cfg3" else (False, True)):
            chunks = (0,) if not a.sweep else (0, 256, 1024, 4096, 16384, 65536, 10 ** 9)
            for ch in chunks:
                lib.proxtv_vjp_tuning(ch)
                ms_b = timed(lambda: bwd(p(y), p(g), p(gx), p(gw) if want_gw else None, B, L, 1, lam, p(w), st), a.steps, a.warmup)
                byts = b * (3 * n + (ne if w is not None else 0) + (ne if want_gw else 0))
                r = {"shape": name, "B": B, "L": L, "dtype": str(x.dtype).replace("torch.", ""), "weighted": w is not None,
                     "gw": want_gw, "chunk": ch, "forward_ms": round(ms_f, 4), "backward_ms": round(ms_b, 4),
                     "backward_GBps": round(byts / ms_b / 1e6, 1), "backward_frac_of_3350": round(byts / ms_b / 1e6 / PEAK_GBS, 3),
                     "backward_faster_than_forward": ms_b < ms_f}
                rows.append(r)
                print(json.dumps(r), flush=True)
            lib.proxtv_vjp_tuning(0)
        del x, w, g, y, gx, gw
        torch.cuda.empty_cache()
    rows.append({"gpu_after": gpu_info()})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
