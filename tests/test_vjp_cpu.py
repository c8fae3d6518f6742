"""CPU tests of the backward pass of the batched 1D TV-L1 prox (proxtv_prox_fibers_vjp_dev_*).

* The math: the host restatement of the contract (vjp_emu.restate) against central finite differences of the oracle's exact prox
  (`port.tv1_linearized`, `port.tv1_weighted`) on signals with well-separated plateaus, where the segmentation is stable under the step:
  J-vector products for gx, the gradient of a scalar penalty, and of per-edge weights (zero weights included, one-sided there).
* The work split changes no bit: the device kernels' chunk scan, carry and fix-up (vjp_core.cuh, run on the host by tests/emu/emu_vjp.cu)
  equal the restatement bit for bit for every chunk length, layout and storage type.
"""
import numpy as np
import pytest

import vjp_emu
from vjp_emu import emulate, restate

CHUNKS = (0, 1, 2, 3, 7, 32, 1000)


@pytest.fixture(scope="module")
def emu():
    return vjp_emu.load()


def plateaus(rng, n, noise=0.05):
    """Levels 3 apart (random order), plateau lengths 3..9, small noise: the prox's segments are the plateaus for lam ~ 0.3."""
    lens = rng.integers(3, 10, n)
    lv = rng.permutation(np.arange(n)) * 3.0
    return (np.repeat(lv, lens) + rng.normal(0, noise, lens.sum()))[:max(lens.sum(), 1)]


def test_restatement_matches_finite_differences_scalar_lambda(port):
    rng = np.random.default_rng(0)
    h = 1e-6
    for trial in range(4):
        x = plateaus(rng, 6)
        lam = 0.3
        y = port.tv1_linearized(x, lam)
        g = rng.normal(0, 1, x.size)
        gx, gw = restate(y[None], g[None], lam)
        gx, gw = gx[0], gw[0]
        # J v by central differences, compared with <gx, v> = <g, J v>
        for _ in range(3):
            v = rng.normal(0, 1, x.size)
            jv = (port.tv1_linearized(x + h * v, lam) - port.tv1_linearized(x - h * v, lam)) / (2 * h)
            assert abs(g @ jv - gx @ v) <= 1e-6 * max(1.0, abs(gx @ v))
        # per-coordinate gradient
        fd = np.array([(g @ port.tv1_linearized(x + h * e, lam) - g @ port.tv1_linearized(x - h * e, lam)) / (2 * h)
                       for e in np.eye(x.size)])
        np.testing.assert_allclose(gx, fd, rtol=1e-6, atol=1e-6)
        # d<g, prox>/d lam = sum of gw
        dl = (g @ port.tv1_linearized(x, lam + h) - g @ port.tv1_linearized(x, lam - h)) / (2 * h)
        assert abs(dl - gw.sum()) <= 1e-6 * max(1.0, abs(dl))


def test_restatement_matches_finite_differences_weights(port):
    rng = np.random.default_rng(1)
    h = 1e-6
    for trial in range(3):
        x = plateaus(rng, 5)
        n = x.size
        w = rng.uniform(0.2, 0.4, n - 1)
        w[rng.choice(n - 1, 4, replace=False)] = 0.0                    # zero-weight edges: never fused
        y = port.tv1_weighted(x, w)
        g = rng.normal(0, 1, n)
        gx, gw = restate(y[None], g[None], 0.0, w[None])
        gx, gw = gx[0], gw[0]
        fd = np.array([(g @ port.tv1_weighted(x + h * e, w) - g @ port.tv1_weighted(x - h * e, w)) / (2 * h) for e in np.eye(n)])
        np.testing.assert_allclose(gx, fd, rtol=1e-6, atol=1e-6)
        f0 = g @ y
        for b in range(n - 1):
            e = np.zeros(n - 1); e[b] = h
            if w[b] == 0:                                                # one-sided: a weight cannot go below 0
                d = (g @ port.tv1_weighted(x, w + e) - f0) / h
            else:
                d = (g @ port.tv1_weighted(x, w + e) - g @ port.tv1_weighted(x, w - e)) / (2 * h)
            assert abs(d - gw[b]) <= 1e-6 * max(1.0, abs(d)), (b, d, gw[b])
        assert np.any(gw[w == 0] != 0)                                   # zero weights did split segments


def test_lambda_zero_is_identity():
    rng = np.random.default_rng(2)
    Y = np.round(rng.normal(0, 1, (3, 50)))                            # equal neighbours: must not be averaged at lam = 0
    G = rng.normal(0, 1, Y.shape)
    gx, gw = restate(Y, G, 0.0)
    assert np.array_equal(gx, G) and np.all(gw[Y[:, 1:] == Y[:, :-1]] == 0)


def cases(rng, dtype):
    """(name, Y, W-or-None, lam): forward-like outputs with ties, runs, constants, ramps, alternation, zero weights."""
    nf, ln = 6, 301
    runs = np.repeat(np.round(rng.normal(0, 2, (nf, ln // 5 + 1))), rng.integers(1, 9, ln // 5 + 1), axis=1)[:, :ln]
    runs = np.concatenate([runs, np.zeros((nf, max(0, ln - runs.shape[1])))], axis=1)
    Wz = rng.uniform(0.1, 1.0, (nf, ln - 1)); Wz[rng.random(Wz.shape) < 0.2] = 0.0
    ramp = np.tile(np.arange(ln, dtype=np.float64), (nf, 1))
    alt = np.where(np.arange(ln) % 2 == 0, 1.0, -1.0)[None, :] * np.ones((nf, 1))
    out = [("runs", runs, None, 0.5), ("runs_zero_w", runs, Wz, 0.0), ("const", np.full((nf, ln), 2.5), None, 1.0),
           ("const_zero_w", np.full((nf, ln), 2.5), Wz, 0.0), ("ramp", ramp, None, 1.0), ("alt", alt, None, 0.3),
           ("offset", 1e6 + runs, None, 1e4), ("lam0", runs, None, 0.0)]
    return [(n, Y.astype(dtype), None if W is None else W.astype(dtype), lam) for n, Y, W, lam in out]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("inc", [1, 3])
def test_chunked_passes_equal_restatement_bit_for_bit(emu, dtype, inc):
    rng = np.random.default_rng(3)
    for name, Y, W, lam in cases(rng, dtype):
        G = rng.normal(0, 1, Y.shape).astype(dtype)
        want_gx, want_gw = restate(Y, G, lam, W)
        for chunk in CHUNKS:
            for want_gw_flag in (True, False):
                gx, gw = emulate(emu, Y, G, lam, W, chunk=chunk, inc=inc, want_gw=want_gw_flag)
                assert np.array_equal(gx, want_gx), (name, chunk)
                if want_gw_flag:
                    assert np.array_equal(gw, want_gw), (name, chunk)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_constant_long_fiber_is_one_carry_chain(emu, dtype):
    """10^5 equal samples: one segment crossing every chunk, so the carry continues one sum through all of them, in order."""
    rng = np.random.default_rng(4)
    Y = np.full((1, 100_000), 0.75, dtype=dtype)
    G = rng.normal(0, 1, Y.shape).astype(dtype)
    want_gx, want_gw = restate(Y, G, 0.5)
    assert np.all(want_gx == want_gx[0, 0]) and np.all(want_gw == 0)
    for chunk in (1, 7, 32, 1000, 4096):
        gx, gw = emulate(emu, Y, G, 0.5, chunk=chunk)
        assert np.array_equal(gx, want_gx) and np.array_equal(gw, want_gw), chunk


def test_chunk_edge_cases(emu):
    """Lengths 1-3, all-singleton ramps and segments ending exactly at chunk boundaries."""
    rng = np.random.default_rng(5)
    for ln in (1, 2, 3, 4, 5, 8, 9):
        for Y in (np.zeros((2, ln)), np.tile(np.arange(ln, dtype=np.float64), (2, 1)), np.repeat(np.arange((ln + 1) // 2), 2)[:ln][None].repeat(2, 0).astype(np.float64)):
            G = rng.normal(0, 1, Y.shape)
            want = restate(Y, G, 0.5)
            for chunk in (1, 2, 3, 4):
                gx, gw = emulate(emu, Y, G, 0.5, chunk=chunk)
                assert np.array_equal(gx, want[0]) and np.array_equal(gw, want[1]), (ln, chunk)
