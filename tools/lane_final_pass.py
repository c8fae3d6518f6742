"""Timeline of the LAST lane launch of a DR2_TV solve (the final projection's row pass): per-task scan / post-scan times, repairs.
usage: lane_final_pass.py [engine]"""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import proxtv_b200 as ptv
import synth_inputs as O
lib = ptv.require_device(); vp = C.c_void_p
lib.proxtv_lane_stats.restype = C.c_ulonglong
eng = sys.argv[1] if len(sys.argv) > 1 else "lane"
maxit = int(sys.argv[2]) if len(sys.argv) > 2 else 0
M = N = 4096
Y = O.gen_cfg2(M, N, seed=0)
y = torch.tensor(np.ascontiguousarray(Y.T), device="cuda").t()      # column-major view
ptv.set_engine(eng)
out = ptv.tv1_2d(y, 0.2, max_iters=maxit); torch.cuda.synchronize()
CAP = 1 << 16
log = torch.zeros(CAP * 16, dtype=torch.int64, device="cuda")      # 16 words per task (proxtv_lane_tasklog)
lib.proxtv_profile_enable(1)                     # plain launches (no graph replay), so that the log pointer is seen
lib.proxtv_lane_stats(1)
lib.proxtv_lane_tasklog(vp(log.data_ptr()), CAP)
out = ptv.tv1_2d(y, 0.2, max_iters=maxit); torch.cuda.synchronize()
lib.proxtv_lane_tasklog(None, 0)
print("repairs in this solve:", lib.proxtv_lane_stats(1))
L = log.cpu().numpy().reshape(-1, 16); L = L[L[:, 0] > 0]
t0 = L[:, 0].min()
start = (L[:, 0] - t0) / 1e3; scan_end = (L[:, 1] - t0) / 1e3; end = (L[:, 2] - t0) / 1e3
print("%d tasks in the log (last launches of the solve overwrite earlier ones; tasks of the final pass: those with the latest start)" % len(L))
late = start > start.max() - 50
print("final pass: %d tasks, span %.1f us; scan median %.1f max %.1f; post (verify + repair) median %.2f p99 %.1f max %.1f us"
      % (late.sum(), end[late].max() - start[late].min(), np.median((scan_end - start)[late]), (scan_end - start)[late].max(),
         np.median((end - scan_end)[late]), np.percentile((end - scan_end)[late], 99), (end - scan_end)[late].max()))
worst = np.argsort((end - scan_end) * late)[-5:]
print("longest post-scan phases (us):", [(int(i), round(float((end - scan_end)[i]), 1)) for i in worst])
