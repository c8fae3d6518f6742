"""CPU tests of the batched weighted 2D prox (tv1w_2d_batched, proxtv_DR2L1W_TV_batched_*; DESIGN.md section 12), no GPU needed.

``forward`` below is drw_device's iteration on a whole batch in storage order: every prox pass runs the oracle's weighted taut string
(``Port.tv1_weighted``, bit-identical to the device's weighted kernels) over the fibers of the batched FiberGeoms -- columns
(N B, M, 1) / rows (M B, N, M) for column-major images, columns (N B, M, N) / rows (M B, N, 1) for C-ordered ones -- with the
weights sliced by the same rule with len - 1 samples per fiber.  It must equal the single-image host forward (drw_vjp_emu.forward)
image by image, bit for bit, in both storage orders, for odd sizes, M == 1 and N == 1: this pins the batch geometry and the weight
layout of include/proxtv_b200.h.  The GPU tests (test_gpu_drw_batched.py) hold the device to this forward and its tapes.

The Python surface checks shapes and weight signs before it touches a device.
"""
import numpy as np
import pytest

import drw_vjp_emu as E
import dr2_vjp_emu as D
from vjp_emu import flat_index


def geoms(M, N, B, row_major):
    """(nf, len, inc) of the column pass (axis 0) and the row pass (axis 1) over B images in storage order."""
    if row_major:
        return (N * B, M, N), (M * B, N, 1)
    return (N * B, M, 1), (M * B, N, M)


def storage(A, row_major):
    """(B, R, C) natural-layout stack -> the flat storage of proxtv_DR2L1W_TV_batched_*: C order, or every image column-major."""
    A = np.asarray(A)
    return np.ascontiguousarray(A if row_major else A.transpose(0, 2, 1)).ravel()


def natural(flat, B, R, C, row_major):
    return flat.reshape(B, R, C) if row_major else flat.reshape(B, C, R).transpose(0, 2, 1)


def fiber_prox(port, y, W, g):
    """The weighted prox of every fiber (nf, len, inc) of the flat array y, weights W (flat, len - 1 samples per fiber)."""
    nf, ln, inc = g
    if ln == 1:
        return y.copy()
    idx, widx = flat_index(nf, ln, inc), flat_index(nf, ln - 1, inc)
    out = np.empty_like(y)
    for f in range(nf):
        out[idx[f]] = port.tv1_weighted(y[idx[f]], W[widx[f]])
    return out


def forward(port, Y, W1, W2, row_major, maxit=0):
    """DR2L1W_TV of the natural-layout stacks Y (B, M, N), W1 (B, M-1, N), W2 (B, M, N-1) in float64, run on their storage (flat);
    returns (out flat, the 2K + 2 flat pass outputs, the two pass geometries, the flat weights).  The start value of each image is
    drw_vjp_emu.forward's (a float64 sum of the image, doubled, divided by M N)."""
    Y = np.asarray(Y, dtype=np.float64)
    B, M, N = Y.shape
    K = E.MAX_ITERS if maxit <= 0 else maxit
    gc, gr = geoms(M, N, B, row_major)
    y, w1, w2 = (storage(np.asarray(A, dtype=np.float64), row_major) for A in (Y, W1, W2))
    t = np.repeat([(2.0 * Y[b].sum()) / float(M * N) for b in range(B)], M * N)
    passes = []
    for k in range(K + 1):
        final = k == K
        x1 = fiber_prox(port, t, w1, gc)
        passes.append(x1)
        d = t - x1
        s = d if final else 2.0 * d - t
        u = y - s
        x2 = fiber_prox(port, u, w2, gr)
        passes.append(x2)
        tw = (u - x2) - y
        if final:
            return -s - tw, passes, (gc, gr), (w1, w2)
        t = 0.5 * (t + (-2.0 * tw - s))


def pass_tapes(passes, geo, w):
    """(F, U) of every flat pass over the whole batch, in storage order (the device tape's passes)."""
    out = []
    for p, X in enumerate(passes):
        nf, ln, inc = geo[p % 2]
        out.append(D.tape_bits(X, nf, ln, inc, 0.0, w[p % 2][flat_index(nf, ln - 1, inc)]))
    return out


def bits(words, n):
    return ((words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(bool).ravel()[:n]


def stack(shape, seed, zeros=0.15):
    """B generic images (blocks plus noise) and weight maps with some zeros, natural layout."""
    B, M, N = shape
    rng = np.random.default_rng(seed)
    Y = np.repeat(np.repeat(rng.normal(0, 1, (B, M // 4 + 1, N // 4 + 1)), 4, axis=1), 4, axis=2)[:, :M, :N] + rng.normal(0, 0.3, shape)
    W1 = rng.uniform(0.05, 0.6, (B, M - 1, N))
    W2 = rng.uniform(0.05, 0.6, (B, M, N - 1))
    W1[rng.random(W1.shape) < zeros] = 0.0
    W2[rng.random(W2.shape) < zeros] = 0.0
    return Y, W1, W2


@pytest.mark.parametrize("row_major", [0, 1])
@pytest.mark.parametrize("shape,maxit", [((3, 7, 9), 2), ((2, 13, 6), 3), ((3, 1, 11), 2), ((3, 10, 1), 2), ((1, 1, 1), 1),
                                         ((2, 9, 9), 35)])
def test_batched_forward_is_the_single_image_forward(port, shape, maxit, row_major):
    B, M, N = shape
    Y, W1, W2 = stack(shape, 11 + M * 7 + N)
    out, passes, geo, w = forward(port, Y, W1, W2, row_major, maxit)
    got = natural(out, B, M, N, row_major)
    tapes = pass_tapes(passes, geo, w)
    assert len(passes) == 2 * maxit + 2
    for b in range(B):
        want, single = E.forward(port, Y[b], W1[b], W2[b], maxit)
        assert np.array_equal(got[b], want), b
        single_tapes = E.pass_tapes(single, W1[b], W2[b])
        for p, X in enumerate(passes):
            assert np.array_equal(natural(X, B, M, N, row_major)[b], single[p]), (b, p)
            # the batch's tapes in storage order are the single image's tapes
            for words, ws in zip(tapes[p], single_tapes[p]):
                assert np.array_equal(natural(bits(words, B * M * N), B, M, N, row_major)[b], bits(ws, M * N).reshape(N, M).T), (b, p)


def test_weight_slicing_matches_the_header_table():
    """The weights of fiber f under the slicing rule are exactly the table of include/proxtv_b200.h for every (b, i, j)."""
    B, M, N = 3, 5, 4
    for row_major in (0, 1):
        gc, gr = geoms(M, N, B, row_major)
        for (nf, ln, inc), (R, Cc), axis in ((gc, (M - 1, N), 0), (gr, (M, N - 1), 1)):
            idx = flat_index(nf, ln - 1, inc)
            flat = np.empty(B * R * Cc, dtype=np.int64)
            flat[idx.ravel()] = np.arange(idx.size)
            assert np.array_equal(np.sort(idx.ravel()), np.arange(B * R * Cc))
            for b in range(B):
                for i in range(R):
                    for j in range(Cc):
                        if row_major:
                            e = b * R * Cc + i * Cc + j
                        else:
                            e = b * R * Cc + j * R + i
                        f, k = divmod(int(flat[e]), ln - 1)
                        # fiber f of image b holds edge k along the pass's axis
                        if axis == 0:
                            assert (f // N, f % N, k) == (b, j, i), (row_major, axis, b, i, j)
                        else:
                            assert (f // M, f % M, k) == (b, i, j), (row_major, axis, b, i, j)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_python_validation_before_any_device_call(dt, monkeypatch):
    import proxtv_b200 as ptv
    monkeypatch.setattr(ptv, "require_device", lambda: (_ for _ in ()).throw(RuntimeError("device reached")))
    x = np.zeros((2, 5, 6), dtype=dt)
    w1, w2 = np.ones((2, 4, 6)), np.ones((2, 5, 5))
    bad = [(x[0], w1[0], w2[0]), (x, w1[:, :3], w2), (x, w1, w2[:, :, :4]), (x, w1[:1], w2), (x, w1, w2[:1]),
           (x, -w1, w2), (x, w1, np.where(np.arange(5) == 2, -1e-9, 1.0) * w2)]
    for a, b, c in bad:
        with pytest.raises(AssertionError):
            ptv.tv1w_2d_batched(a, b, c)
