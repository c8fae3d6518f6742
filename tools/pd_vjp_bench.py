"""Times of the PD_TV and PD2_TV backward passes (DESIGN.md section 14) against the no-grad solve (CUDA events, warmup, device-resident
buffers):

  vol-f32   PD_TV on one 512 x 512 x 256 float32 volume (BASELINE config 4's), column-major, 3 terms ws = (0.2, 0.2, 0.2) on axes
            (1, 2, 3)
  4k-f64    PD2_TV on one 4096 x 4096 float64 image (BASELINE config 2's kind), column-major, 2 terms ws = (0.2, 0.2) on axes (1, 2)

maxIters 0 (35; the stop rule may end a solve earlier: the iteration count run is reported).  For each: the no-grad solve
(proxtv_PD*_TV_dev_*), the recorded forward (proxtv_PD*_TV_record_dev_*), the backward without and with the penalty gradients
(proxtv_PD*_TV_vjp_dev_*), and the tape's size.  Prints one JSON line per shape and the card's name, power limit and SM clock before
and after (read-only nvidia-smi query).  Changes no device setting.

    python tools/pd_vjp_bench.py [--steps 5] [--warmup 1] [--out FILE]
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
import synth_inputs as S  # noqa: E402
from dr2_vjp_bench import gpu_info, p, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = ptv.require_device()
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    for name, shape, dt, ws in (("vol-f32", (512, 512, 256), torch.float32, [0.2, 0.2, 0.2]),
                                ("4k-f64", (4096, 4096), torch.float64, [0.2, 0.2])):
        solver = "PD2_TV" if len(ws) == 2 else "PD_TV"                       # tvgen's dispatch
        f32 = dt == torch.float32
        V = S.gen_cfg4(shape, seed=0) if len(shape) == 3 else S.gen_cfg2(*shape, seed=0)
        Y = torch.from_numpy(np.ascontiguousarray(V.ravel(order="F"))).to(device="cuda", dtype=dt)   # the column-major buffer
        del V
        out, G, gY = torch.empty_like(Y), torch.randn_like(Y), torch.empty_like(Y)
        npen = len(ws)
        ns = np.array(shape, dtype=np.int32)
        dims = np.arange(1, npen + 1, dtype=np.float64)
        lam = np.array(ws, dtype=np.float64)
        glam = torch.empty(npen, dtype=torch.float64, device="cuda")
        nb = getattr(lib, "proxtv_%s_tape_bytes" % solver)(p_np(ns), len(shape), npen, 0)
        tape = torch.empty(nb, dtype=torch.uint8, device="cuda")
        info = np.zeros(3)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        sfx = "f32" if f32 else "f64"
        solve = getattr(lib, "proxtv_%s_dev_%s" % (solver, sfx))
        rec = getattr(lib, "proxtv_%s_record_dev_%s" % (solver, sfx))
        vjp = getattr(lib, "proxtv_%s_vjp_dev_%s" % (solver, sfx))
        ip = p_np(info)

        def lam_p():                      # PD_TV scales the penalties in place: fresh values each time
            lam[:] = ws
            return p_np(lam)
        ms_solve = timed(lambda: solve(p(Y), lam_p(), p_np(dims), p(out), ip, p_np(ns), len(shape), npen, 0, st), a.steps, a.warmup)
        ref, ref_info = out.clone(), info.copy()
        ms_rec = timed(lambda: rec(p(Y), lam_p(), p_np(dims), p(out), ip, p_np(ns), len(shape), npen, 0, p(tape), nb, st),
                       a.steps, a.warmup)
        same = bool(torch.equal(out, ref)) and bool(np.array_equal(info, ref_info))
        K = int(info[0])
        ms_b = timed(lambda: vjp(p_np(ns), len(shape), npen, p_np(dims), 0, K, p(tape), p(G), p(gY), None, st), a.steps, a.warmup)
        ms_bw = timed(lambda: vjp(p_np(ns), len(shape), npen, p_np(dims), 0, K, p(tape), p(G), p(gY), p(glam), st), a.steps, a.warmup)
        r = {"shape": name, "solver": solver, "dims": list(shape), "terms": npen, "iterations": K, "dtype": str(dt).replace("torch.", ""), "solve_ms": round(ms_solve, 3),
             "record_ms": round(ms_rec, 3), "backward_ms": round(ms_b, 3), "backward_glam_ms": round(ms_bw, 3),
             "tape_MiB": round(nb / 2 ** 20, 1), "record_equals_solve": same}
        rows.append(r)
        print(json.dumps(r), flush=True)
        del Y, out, ref, G, gY, glam, tape
        torch.cuda.empty_cache()
        lib.proxtv_release_workspace()
    rows.append({"gpu_after": gpu_info()})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


def p_np(a):
    return C.c_void_p(a.ctypes.data)


if __name__ == "__main__":
    main()
