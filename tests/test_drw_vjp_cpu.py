"""CPU tests of the DR2L1W_TV backward pass (DESIGN.md section 12), no GPU needed.

The host restatement (drw_vjp_emu.backward) is the exact derivative of the host forward (drw_vjp_emu.forward: drw_device's iteration
on the oracle's weighted taut string): gY, gW1 and gW2 agree with finite differences to 1e-6 relative -- element by element for every
input and every weight on 6 x 7 and 9 x 5 images, along random directions on 40 x 56, for 1, 2, 5 and 35 iterations, and with M == 1
and N == 1.  Zero weights are included; the prox is defined for weights >= 0 only, so theirs is the right derivative (forward
differences).  The unrolled map is piecewise linear, so each difference is taken at the largest step from 1e-6 down that holds no
kink (its two estimates agree).  The tape-driven form of the restatement (backward_from_tapes) equals the pass-driven one bit for bit.
"""
import numpy as np
import pytest

import drw_vjp_emu as E

EPS = 1e-6


def image(shape, seed):
    """Blocks plus noise: generic data (no ties in the input), so the segmentations are locally constant around it."""
    rng = np.random.default_rng(seed)
    M, N = shape
    return np.repeat(np.repeat(rng.normal(0, 1, (M // 4 + 1, N // 4 + 1)), 4, axis=0), 4, axis=1)[:M, :N] + rng.normal(0, 0.3, shape)


def weights(shape, seed, zeros=0.15):
    rng = np.random.default_rng(seed)
    M, N = shape
    W1 = rng.uniform(0.1, 0.5, (M - 1, N))
    W2 = rng.uniform(0.1, 0.5, (M, N - 1))
    W1[rng.random(W1.shape) < zeros] = 0.0
    W2[rng.random(W2.shape) < zeros] = 0.0
    return W1, W2


def objective(port, Y, W1, W2, G, maxit):
    return float(np.sum(E.forward(port, Y, W1, W2, maxit)[0] * G))


def check_close(fd, an, tol=1e-6):
    fd, an = np.asarray(fd, dtype=np.float64), np.asarray(an, dtype=np.float64)
    scale = max(np.max(np.abs(an)) if an.size else 0.0, 1e-300)
    assert np.max(np.abs(fd - an), initial=0.0) <= tol * scale, (np.max(np.abs(fd - an)) / scale, fd.ravel()[:6], an.ravel()[:6])


def kink_free(step, eps_list=(EPS, 1e-7, 1e-8)):
    """Difference quotient of a piecewise linear function of one step size (step(e) -> f(x + e) - f(x)) at the first step whose two
    estimates agree to 1e-6 -- the two one-sided quotients, or, for a right derivative (step(-e) is None), the quotients at e and e / 2
    -- i.e. no segment merges or splits within the step.  Below 1e-8 rounding takes over."""
    for eps in eps_list:
        p = step(eps) / eps
        m = step(-eps)
        q = (step(eps / 2) / (eps / 2)) if m is None else -m / eps
        if abs(p - q) <= 1e-6 * max(abs(p), abs(q), 1.0):
            return p if m is None else (p + q) / 2
    raise AssertionError("every step crosses a kink")


def fd_elementwise(port, Y, W1, W2, G, maxit):
    """Finite differences of the objective for every entry of Y, W1, W2: central, one-sided (right) for a weight at 0."""
    f = lambda args: objective(port, *args, G, maxit)          # noqa: E731
    f0 = f((Y, W1, W2))
    out = []
    for which in range(3):
        A = (Y, W1, W2)[which]
        fd = np.empty_like(A)
        for idx in np.ndindex(*A.shape):
            right = which > 0 and A[idx] == 0.0

            def step(e):
                if right and e < 0:
                    return None
                Ae = A.copy(); Ae[idx] += e
                args = [Y, W1, W2]; args[which] = Ae
                return f(args) - f0
            fd[idx] = kink_free(step)
        out.append(fd)
    return out


@pytest.mark.parametrize("shape", [(6, 7), (9, 5)], ids=["6x7", "9x5"])
@pytest.mark.parametrize("maxit", [1, 2, 5, 35])
def test_elementwise(port, shape, maxit):
    Y = image(shape, 11 + maxit)
    W1, W2 = weights(shape, 3 + maxit)
    assert (W1 == 0).any() and (W2 == 0).any()
    G = np.random.default_rng(5).normal(size=shape)
    _, passes = E.forward(port, Y, W1, W2, maxit)
    gY, gW1, gW2 = E.backward(passes, G, W1, W2, maxit)
    fY, f1, f2 = fd_elementwise(port, Y, W1, W2, G, maxit)
    check_close(fY, gY)
    check_close(f1, gW1)
    check_close(f2, gW2)


@pytest.mark.parametrize("maxit", [1, 2, 5, 35])
def test_directional(port, maxit):
    """40 x 56: random directions in Y and in each weight map on its own (directions vanish on the zero weights, whose derivative is
    one-sided and checked element by element above)."""
    shape = (40, 56)
    Y = image(shape, 3 + maxit)
    W1, W2 = weights(shape, 7 + maxit)
    rng = np.random.default_rng(17)
    G = rng.normal(size=shape)
    _, passes = E.forward(port, Y, W1, W2, maxit)
    gY, gW1, gW2 = E.backward(passes, G, W1, W2, maxit)
    f0 = objective(port, Y, W1, W2, G, maxit)
    V = rng.normal(size=shape)
    check_close([kink_free(lambda e: objective(port, Y + e * V, W1, W2, G, maxit) - f0)], [np.sum(gY * V)])
    V1 = rng.normal(size=W1.shape) * (W1 > 0)
    check_close([kink_free(lambda e: objective(port, Y, W1 + e * V1, W2, G, maxit) - f0)], [np.sum(gW1 * V1)])
    V2 = rng.normal(size=W2.shape) * (W2 > 0)
    check_close([kink_free(lambda e: objective(port, Y, W1, W2 + e * V2, G, maxit) - f0)], [np.sum(gW2 * V2)])


@pytest.mark.parametrize("shape", [(1, 9), (8, 1)], ids=["M1", "N1"])
def test_single_row_and_column(port, shape):
    """M == 1 / N == 1: the length-1 fibers are the identity, and that weight map is empty."""
    Y = image(shape, 2)
    W1, W2 = weights(shape, 4)
    G = np.random.default_rng(1).normal(size=shape)
    _, passes = E.forward(port, Y, W1, W2, 3)
    gY, gW1, gW2 = E.backward(passes, G, W1, W2, 3)
    assert gW1.shape == W1.shape and gW2.shape == W2.shape
    fY, f1, f2 = fd_elementwise(port, Y, W1, W2, G, 3)
    check_close(fY, gY)
    check_close(f1, gW1)
    check_close(f2, gW2)


@pytest.mark.parametrize("shape", [(6, 7), (40, 56), (1, 9), (8, 1)])
@pytest.mark.parametrize("maxit", [2, 35])
def test_tape_driven_restatement_equals_pass_driven(port, shape, maxit):
    Y = np.round(image(shape, 9) * 4) / 4                # ties in the input: segments with zero-weight equal edges appear
    W1, W2 = weights(shape, 5, zeros=0.3)
    G = np.random.default_rng(2).normal(size=shape)
    _, passes = E.forward(port, Y, W1, W2, maxit)
    want = E.backward(passes, G, W1, W2, maxit)
    got = E.backward_from_tapes(E.pass_tapes(passes, W1, W2), G, maxit)
    for a, b in zip(got, want):
        assert a.shape == b.shape and np.array_equal(a, b)
    G32, passes32 = G.astype(np.float32), [X.astype(np.float32) for X in passes]
    got32 = E.backward_from_tapes(E.pass_tapes(passes32, W1, W2), G32, maxit)
    want32 = E.backward(passes32, G32, W1, W2, maxit)
    for a, b in zip(got32, want32):
        assert a.dtype == np.float32 and np.array_equal(a, b)
