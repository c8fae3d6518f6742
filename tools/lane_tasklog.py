"""Per-task log of the three lane passes of a DR2_TV solve on the config-2 image (4096^2 f64), at a mid-solve iterate: the column pass
(k_lane<CONTIG, plain>), the staged row pass (<STRIDED, LOP_DR_B>) and the final row pass (<STRIDED, LOP_DR_B_FINAL>).  Per pass: the
timeline (when tasks start / end, tail), and where each warp's cycles go (include/proxtv_b200.h: proxtv_lane_tasklog).
usage: lane_tasklog.py [iterations before the logged passes, default 17] [variant] [clen]"""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import proxtv_b200 as ptv
import synth_inputs as O
lib = ptv.require_device(); vp = C.c_void_p
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 17
variant = int(sys.argv[2]) if len(sys.argv) > 2 else 0
clen = int(sys.argv[3]) if len(sys.argv) > 3 else 0
LANE_PLAIN, LANE_DR_B, LANE_DR_B_FINAL = 0, 1, 2
WORDS = 16
M = N = 4096
LAM = 0.2
Y = O.gen_cfg2(M, N, seed=0)
y = torch.tensor(np.ascontiguousarray(Y.T), device="cuda")        # column-major image: row j of y = column j of Y
t = torch.full_like(y, 2.0 * float(y.mean()))                     # the solver's start value (solver.cu: dr2_lane_body)
x1 = torch.empty_like(y); t2 = torch.empty_like(y); out = torch.empty_like(y)
lib.proxtv_lane_tuning(clen, 32, variant)
st = vp(torch.cuda.current_stream().cuda_stream)


def col_pass():      # x1 = prox_cols(t): N contiguous fibers of length M
    assert lib.proxtv_lane_prox_dev_f64(LANE_PLAIN, vp(t.data_ptr()), None, None, vp(x1.data_ptr()), N, M, 1, LAM, st), lib.proxtv_last_error()


def row_pass(final):  # t2 = (t - x1) + prox_rows(Y - (2 (t - x1) - t)), or out = prox_rows(Y - (t - x1)): M fibers of length N, stride M
    assert lib.proxtv_lane_prox_dev_f64(LANE_DR_B_FINAL if final else LANE_DR_B, vp(y.data_ptr()), vp(x1.data_ptr()), vp(t.data_ptr()),
                                        vp((out if final else t2).data_ptr()), M, N, M, LAM, st), lib.proxtv_last_error()


for _ in range(iters):
    col_pass(); row_pass(False); t, t2 = t2, t
torch.cuda.synchronize()
CAP = 1 << 16
log = torch.zeros(CAP * WORDS, dtype=torch.int64, device="cuda")


def logged(name, fn):
    log.zero_()
    lib.proxtv_lane_tasklog(vp(log.data_ptr()), CAP)
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    lib.proxtv_lane_tasklog(None, 0)
    L = log.cpu().numpy().reshape(-1, WORDS)
    L = L[L[:, 0] > 0]
    report(name, L, e0.elapsed_time(e1) * 1e3)


def q(v):
    return "%8.0f %8.0f %8.0f" % (np.percentile(v, 10), np.median(v), np.percentile(v, 90))


def report(name, L, event_us):
    nt = len(L)
    t0 = L[:, 0].min()
    start = (L[:, 0] - t0) / 1e3; scan_end = (L[:, 1] - t0) / 1e3; end = (L[:, 2] - t0) / 1e3; sm = L[:, 3]
    print("== %s: %d tasks, event time %.1f us, log span %.1f us (variant %d, after %d iterations)" % (name, nt, event_us, end.max(), variant, iters))
    dur = scan_end - start
    print("scan   : min %.1f  p10 %.1f  median %.1f  p90 %.1f  max %.1f us" % (dur.min(), np.percentile(dur, 10), np.median(dur), np.percentile(dur, 90), dur.max()))
    print("scanend: min %.1f  p10 %.1f  median %.1f  p90 %.1f  max %.1f us" % (scan_end.min(), np.percentile(scan_end, 10), np.median(scan_end), np.percentile(scan_end, 90), scan_end.max()))
    post = end - scan_end
    print("post   : median %.2f  p99 %.1f  max %.1f us   (records, verification, repairs)" % (np.median(post), np.percentile(post, 99), post.max()))
    per_sm = np.bincount(sm.astype(int), minlength=132)       # H100 SXM: 132 SMs
    print("tasks per SM: min %d max %d" % (per_sm.min(), per_sm.max()))
    T = end.max(); area = np.sum(end - start)
    print("mean residency %.1f%% of %d tasks x span (tail loss %.1f%%)" % (100 * area / (nt * T), nt, 100 - 100 * area / (nt * T)))
    epochs, steps, starved, waits, cyc = L[:, 4], L[:, 5], L[:, 6], L[:, 7], L[:, 8].astype(np.float64)
    rows = L[:, 14].astype(np.float64)
    parts = {"tile wait": L[:, 9], "no-move other": L[:, 10], "sweep+drain": L[:, 11], "feed": L[:, 12], "scan": L[:, 13]}
    parts["reductions"] = cyc - sum(v.astype(np.float64) for v in parts.values())
    print("per task                          p10   median      p90")
    print("  rows scanned               %s" % q(rows))
    print("  epochs                     %s" % q(epochs))
    print("  scan steps                 %s" % q(steps))
    print("  steps per epoch            %s" % q(steps / np.maximum(epochs, 1)))
    print("  starved epochs (< 8 steps) %s" % q(starved))
    print("  tile waits                 %s" % q(waits))
    print("  cycles                     %s" % q(cyc))
    print("  cycles per row             %s" % q(cyc / rows))
    print("share of the epoch loop's cycles (sum over tasks) and cycles per row (median task):")
    for k, v in parts.items():
        print("  %-14s %5.1f%%  %7.0f cycles/row" % (k, 100 * v.sum() / cyc.sum(), np.median(v / rows)))


logged("column pass  k_lane<CONTIG, plain>", col_pass)
logged("row pass     k_lane<STRIDED, LOP_DR_B>", lambda: row_pass(False))
logged("final pass   k_lane<STRIDED, LOP_DR_B_FINAL>", lambda: row_pass(True))
