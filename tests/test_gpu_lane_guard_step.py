"""The lane guard's mean step (elementwise.cu: ew_mean_abs_step) is pinned bit for bit to its summation order: the terms
|y[e + 1] - y[e]| of e = j, j + 256, ... summed in that order into s_j, the 256 sums combined by a pairwise tree, divided by n - 1.
The guard takes the lane engine iff lam <= kappa * step (kappa 1 float64, 2 float32), so a solve under engine 'auto' with lam at the
last representable value on either side of kappa * step shows the device's step exactly (proxtv_lane_guard_last)."""
import ctypes as C

import numpy as np
import pytest


def exact_step(flat):
    """solver.cu lane_guard: the mean step over the first 2^18 stored elements, in the device's summation order."""
    ns = min(flat.size, 1 << 18)
    y = flat[:ns].astype(np.float64)
    terms = np.abs(y[1:] - y[:-1])
    k = -(-terms.size // 256)
    t = np.zeros(k * 256)               # lanes past the last term add +0.0: the sums do not change
    t[:terms.size] = terms
    t = t.reshape(k, 256)
    s = np.zeros(256)
    for r in range(k):                  # lane j: its terms in increasing e
        s = s + t[r]
    w = 128
    while w > 0:                        # sh[j] += sh[j + w]
        s[:w] = s[:w] + s[w:2 * w]
        w //= 2
    return s[0] / (ns - 1)


CASES = [(np.float64, 600, 500, 0), (np.float64, 64, 48, 1), (np.float64, 3, 50, 2), (np.float32, 512, 700, 3), (np.float32, 40, 40, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,M,N,seed", CASES, ids=["%s-%dx%d" % (np.dtype(c[0]).name, c[1], c[2]) for c in CASES])
def test_guard_step_is_exact(ptv, dt, M, N, seed):
    import torch
    lib = ptv.load()
    rng = np.random.default_rng(seed)
    flat = (np.cumsum(rng.normal(0, 1, M * N)) * 0.1 + rng.normal(0, 0.5, M * N)).astype(dt)     # stored order: column-major M x N
    kappa = 1.0 if dt == np.float64 else 2.0
    thr = kappa * exact_step(flat)
    assert thr > 0
    if dt == np.float64:
        below, above = thr, np.nextafter(thr, np.inf)
    else:
        below = np.float32(thr)
        if float(below) > thr:
            below = np.nextafter(below, np.float32(0))
        above = np.nextafter(below, np.float32(np.inf))
    assert float(below) <= thr < float(above)
    tdt = torch.float64 if dt == np.float64 else torch.float32
    Y = torch.from_numpy(flat).to(device="cuda", dtype=tdt)
    out = torch.empty_like(Y)
    fn = lib.proxtv_DR2_TV_dev_f64 if dt == np.float64 else lib.proxtv_DR2_TV_dev_f32
    prev = ptv.set_engine("auto")
    try:
        for lam, want in ((below, 1), (above, 0)):
            info = np.zeros(3)
            fn(M, N, 1, 0, C.c_void_p(Y.data_ptr()), float(lam), float(lam), C.c_void_p(out.data_ptr()), 2, C.c_void_p(info.ctypes.data), None)
            torch.cuda.synchronize()
            assert lib.proxtv_lane_guard_last() == want, (float(lam), thr)
    finally:
        ptv.set_engine(prev)
