"""CPU tests of the DR2_TV backward pass (DESIGN.md section 11), no GPU needed.

* The host restatement (dr2_vjp_emu.backward) is the exact derivative of the host forward (dr2_vjp_emu.forward: the lane schedule on
  the sequential slope-form scan): it agrees with central differences to 1e-6 relative -- element by element on tiny images, along
  random directions on larger batches, for both penalties separately, and for 1, 2, 5 and 35 iterations.
* The tape-driven chunk logic of the backward kernels (vjp_core.cuh: VjpScan::step, vjp_fix_chunk_sg), compiled with g++, equals the
  y-driven one (vjp_emu.emulate, itself pinned to the restatement by test_vjp_cpu.py) bit for bit, and the encoder (vjp_tape_edge)
  equals the numpy tape.
"""
import numpy as np
import pytest

import dr2_vjp_emu as D
import lane_emu
import vjp_emu


@pytest.fixture(scope="module")
def emu():
    return lane_emu.load()


def images(shape, seed):
    """Blocks plus noise: generic data (no ties in the input), so the segmentations are locally constant around it."""
    rng = np.random.default_rng(seed)
    B, M, N = shape
    return np.repeat(np.repeat(rng.normal(0, 1, (B, M // 4 + 1, N // 4 + 1)), 4, axis=1), 4, axis=2)[:, :M, :N] + rng.normal(0, 0.3, shape)


def objective(emu, Y, G, w1, w2, maxit):
    return float(np.sum(D.forward(emu, Y, w1, w2, maxit)[0] * G))


def check_close(fd, an, tol=1e-6):
    fd, an = np.asarray(fd, dtype=np.float64), np.asarray(an, dtype=np.float64)
    scale = max(np.max(np.abs(an)), 1e-300)
    assert np.max(np.abs(fd - an)) <= tol * scale, (np.max(np.abs(fd - an)) / scale, fd.ravel()[:6], an.ravel()[:6])


@pytest.mark.parametrize("shape", [(1, 6, 7), (2, 9, 5)], ids=["6x7", "2x9x5"])
@pytest.mark.parametrize("maxit", [1, 2, 5, 35])
def test_gY_elementwise(emu, shape, maxit):
    Y = images(shape, 11 + maxit)
    G = np.random.default_rng(5).normal(size=shape)
    w1, w2 = 0.25, 0.35
    _, passes = D.forward(emu, Y, w1, w2, maxit)
    gY, _ = D.backward(passes, G, w1, w2, maxit)
    eps = 1e-6
    fd = np.empty_like(Y)
    for idx in np.ndindex(*shape):
        Yp = Y.copy(); Yp[idx] += eps
        Ym = Y.copy(); Ym[idx] -= eps
        fd[idx] = (objective(emu, Yp, G, w1, w2, maxit) - objective(emu, Ym, G, w1, w2, maxit)) / (2 * eps)
    check_close(fd, gY)


@pytest.mark.parametrize("maxit", [1, 2, 5, 35])
def test_directional_and_penalties(emu, maxit):
    """40 x 56 batch of 2: random directions in Y, and each penalty on its own with W1 != W2 (the gradient of a penalty is the sum of
    glam over images; per image too, since the images are independent)."""
    shape = (2, 40, 56)
    Y = images(shape, 3 + maxit)
    rng = np.random.default_rng(17)
    G = rng.normal(size=shape)
    w1, w2 = 0.2, 0.45
    _, passes = D.forward(emu, Y, w1, w2, maxit)
    gY, glam = D.backward(passes, G, w1, w2, maxit)
    eps = 1e-6
    for _ in range(2):
        V = rng.normal(size=shape)
        fd = (objective(emu, Y + eps * V, G, w1, w2, maxit) - objective(emu, Y - eps * V, G, w1, w2, maxit)) / (2 * eps)
        check_close([fd], [np.sum(gY * V)])
    for b in range(2):
        Yb, Gb = Y[b:b + 1], G[b:b + 1]
        fd1 = (objective(emu, Yb, Gb, w1 + eps, w2, maxit) - objective(emu, Yb, Gb, w1 - eps, w2, maxit)) / (2 * eps)
        fd2 = (objective(emu, Yb, Gb, w1, w2 + eps, maxit) - objective(emu, Yb, Gb, w1, w2 - eps, maxit)) / (2 * eps)
        check_close([fd1], [glam[b, 0]])
        check_close([fd2], [glam[b, 1]])


def test_single_row_and_column(emu):
    """M == 1 (the start image's column prox is the identity) and N == 1."""
    for shape in ((1, 1, 9), (1, 8, 1)):
        Y = images(shape, 2)
        G = np.random.default_rng(1).normal(size=shape)
        _, passes = D.forward(emu, Y, 0.3, 0.3, 3)
        gY, _ = D.backward(passes, G, 0.3, 0.3, 3)
        eps = 1e-6
        fd = np.empty_like(Y)
        for idx in np.ndindex(*shape):
            Yp = Y.copy(); Yp[idx] += eps
            Ym = Y.copy(); Ym[idx] -= eps
            fd[idx] = (objective(emu, Yp, G, 0.3, 0.3, 3) - objective(emu, Ym, G, 0.3, 0.3, 3)) / (2 * eps)
        check_close(fd, gY)


# ---------------------------------------------------------------------------------------------------------------- tape-driven chunk logic
def fibers(kind, nf, ln, rng):
    if kind == "blocks":
        return np.repeat(rng.normal(0, 1, (nf, ln // 7 + 1)), 7, axis=1)[:, :ln]
    if kind == "ties":
        return np.round(rng.normal(0, 1.5, (nf, ln)))
    if kind == "const":
        return np.full((nf, ln), 0.75)
    raise ValueError(kind)


def tape_of(vemu, Y, inc, lam, W):
    """(F, U) of the fibers Y (nf, ln) laid out with stride inc, from the g++ encoder; checked against the numpy tape."""
    nf, ln = Y.shape
    y = vjp_emu.to_flat(Y, inc)
    nw = D.tape_words(nf * ln)
    F = np.full(nw, 0xdeadbeef, dtype=np.uint32); U = F.copy()
    w = vjp_emu.to_flat(np.ascontiguousarray(W, dtype=Y.dtype), inc) if W is not None else None
    fn = vemu.emu_tape_f32 if Y.dtype == np.float32 else vemu.emu_tape_f64
    fn(y.ctypes.data, nf, ln, inc, Y.dtype.type(lam), w.ctypes.data if w is not None else None, F.ctypes.data, U.ctypes.data)
    Fn, Un = D.tape_bits(y, nf, ln, inc, lam, W)
    assert np.array_equal(F, Fn) and np.array_equal(U, Un)
    return F, U


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_tape_chunk_logic_equals_y_driven(dt):
    yemu, vemu = vjp_emu.load(), D.load()
    rng = np.random.default_rng(23)
    cases = 0
    for kind in ("blocks", "ties", "const"):
        for nf, ln, inc in ((6, 1000, 1), (4, 333, 4), (3, 1, 1), (5, 2, 5)):
            Y = fibers(kind, nf, ln, rng).astype(dt)
            G = rng.normal(size=(nf, ln)).astype(dt)
            W = np.where(rng.random((nf, max(ln - 1, 0))) < 0.2, 0.0, 1.0).astype(dt)     # zero weights: equal but not fused
            for lam, Wx in ((0.5, None), (0.0, None), (0.0, W)):
                F, U = tape_of(vemu, Y, inc, lam, Wx)
                for chunk in (0, 1, 2, 3, 7, 32, 100, 999, 1000):
                    want = vjp_emu.emulate(yemu, Y, G, lam, Wx, chunk=chunk, inc=inc)
                    got = D.emulate_tape(vemu, F, U, G, nf, ln, inc, chunk=chunk)
                    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (kind, nf, ln, inc, lam, chunk)
                    cases += 1
    # every chunk length 1..1000 on one mixed fiber
    Y = np.concatenate([fibers("ties", 1, 500, rng), fibers("const", 1, 500, rng)], axis=1).astype(dt)
    G = rng.normal(size=Y.shape).astype(dt)
    F, U = tape_of(vemu, Y, 1, 0.3, None)
    for chunk in range(1, 1001):
        want = vjp_emu.emulate(yemu, Y, G, 0.3, chunk=chunk)
        got = D.emulate_tape(vemu, F, U, G, 1, 1000, 1, chunk=chunk)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), chunk
    assert cases > 0


def test_tape_constant_long_fiber():
    """A constant 10^5-sample fiber: one segment through every chunk (one sequential chain in pass 2)."""
    yemu, vemu = vjp_emu.load(), D.load()
    ln = 100000
    Y = np.full((1, ln), 1.5)
    G = np.random.default_rng(4).normal(size=(1, ln))
    F, U = tape_of(vemu, Y, 1, 0.2, None)
    for chunk in (0, 256, 4096):
        want = vjp_emu.emulate(yemu, Y, G, 0.2, chunk=chunk)
        got = D.emulate_tape(vemu, F, U, G, 1, ln, 1, chunk=chunk)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), chunk
