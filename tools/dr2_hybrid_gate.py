"""Column pass of a DR2_TV solve on a column-major 4096^2 float64 image, timed both ways the lane engine can run it:
    CONTIG   k_lane<CONTIG, LOP_PLAIN>     over the column-major array (N contiguous fibers of length M; TMA box in, TMA box out)
    PLAIN_T  k_lane<STRIDED, LOP_PLAIN_T>  over its row-major transpose (fibers of stride N; result written transposed, i.e. column-major)
on bench's config-2 image and on a real iterate t (the staged schedule stopped after `iters` iterations).  Both must give the same x1
bit for bit.  For the row pass, the cost of a transposed drain: k_lane<STRIDED, LOP_PLAIN> against <STRIDED, LOP_PLAIN_T> over the
rows of the column-major image, and the staged row pass k_lane<STRIDED, LOP_DR_B> itself.
This decides whether keeping the iterate row-major can pay (DESIGN.md section 6): the column pass must save more per launch than the
row pass's transposed drain costs, which at 4096^2 means well over 20 us at the iterate.  It did not (H100, 700 W: +2.3 us).
usage: dr2_hybrid_gate.py [iterations before the iterate, default 17] [timed launches, default 50] [JSON file for the results]"""
import ctypes as C, json, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import proxtv_b200 as ptv
import synth_inputs as O

LANE_PLAIN, LANE_DR_B, LANE_PLAIN_T = 0, 1, 6
M = N = 4096
LAM = 0.2
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 17
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 50
json_out = sys.argv[3] if len(sys.argv) > 3 else None
lib = ptv.require_device(); vp = C.c_void_p
lib.proxtv_lane_prox_dev_f64.argtypes = [C.c_int, vp, vp, vp, vp, C.c_longlong, C.c_int, C.c_longlong, C.c_double, vp]
st = vp(torch.cuda.current_stream().cuda_stream)
p = lambda a: vp(a.data_ptr()) if a is not None else None        # noqa: E731


def lane(op, A, B, Cc, X, nf, ln, inc):
    assert lib.proxtv_lane_prox_dev_f64(op, p(A), p(B), p(Cc), p(X), nf, ln, inc, LAM, st) == 1, lib.proxtv_last_error()


def timeit(fn):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3       # us per launch


def smi():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi: %s" % e


y = torch.tensor(np.ascontiguousarray(O.gen_cfg2(M, N, seed=0).T), device="cuda")   # column-major image: row j of y = column j of Y
# a real iterate: the staged schedule (solver.cu: dr2_lane_body) run by hand for `iters` iterations
t = torch.full_like(y, 2.0 * float(y.mean())); x1 = torch.empty_like(y); t2 = torch.empty_like(y)
for it in range(iters):
    if it: lane(LANE_PLAIN, t, None, None, x1, N, M, 1)
    lane(LANE_DR_B, y, t if it == 0 else x1, t, t2, M, N, M)
    t, t2 = t2, t
torch.cuda.synchronize()

OUT = {"gpu": smi(), "iters": iters, "reps": reps, "col": {}, "row": {}}
bytes_col = 2 * M * N * 8
xc = torch.empty_like(y); xt = torch.empty_like(y)
for name, a in (("cfg2_image", y), ("iterate_%d" % iters, t)):
    ar = a.t().contiguous()                                        # row-major copy: (M, N), column j strided by N
    lane(LANE_PLAIN, a, None, None, xc, N, M, 1)
    lane(LANE_PLAIN_T, ar, None, None, xt, N, M, N)
    torch.cuda.synchronize()
    same = bool(torch.equal(xc, xt))
    us_c = timeit(lambda: lane(LANE_PLAIN, a, None, None, xc, N, M, 1))
    us_t = timeit(lambda: lane(LANE_PLAIN_T, ar, None, None, xt, N, M, N))
    OUT["col"][name] = dict(contig_us=us_c, plain_t_us=us_t, saving_us=us_c - us_t, contig_tbs=bytes_col / us_c / 1e6,
                            plain_t_tbs=bytes_col / us_t / 1e6, bit_identical=same)
    print("column pass, %-12s CONTIG %7.1f us (%.2f TB/s)   PLAIN_T %7.1f us (%.2f TB/s)   saving %6.1f us   x1 identical: %s"
          % (name, us_c, bytes_col / us_c / 1e6, us_t, bytes_col / us_t / 1e6, us_c - us_t, same), flush=True)
# row pass at the iterate: the price of a transposed drain, and the staged row pass itself
lane(LANE_PLAIN, t, None, None, x1, N, M, 1)
u = (y - (2 * (t - x1) - t)).contiguous()
us_s = timeit(lambda: lane(LANE_PLAIN, u, None, None, xc, M, N, M))
us_st = timeit(lambda: lane(LANE_PLAIN_T, u, None, None, xt, M, N, M))
us_b = timeit(lambda: lane(LANE_DR_B, y, x1, t, t2, M, N, M))
OUT["row"] = dict(strided_plain_us=us_s, strided_plain_t_us=us_st, transposed_drain_us=us_st - us_s, dr_b_us=us_b)
print("row pass at the iterate: STRIDED PLAIN %.1f us, PLAIN_T %.1f us (transposed drain +%.1f us); staged DR_B %.1f us"
      % (us_s, us_st, us_st - us_s, us_b), flush=True)
OUT["gpu_after"] = smi()
print(OUT["gpu"], "|", OUT["gpu_after"])
if json_out:
    with open(json_out, "w") as f:
        json.dump(OUT, f, indent=1)
