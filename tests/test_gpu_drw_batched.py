"""GPU tests (-m gpu) of the batched weighted 2D prox: proxtv_DR2L1W_TV_batched_* (DESIGN.md section 12) and tv1w_2d_batched.

Bars:
  * forward: every image of a batch == proxtv_DR2L1W_TV_dev_* on that image, bit for bit, on dyadic inputs with some zero weights
    (their sums are exact, so the start value does not depend on how the per-image reduction is split) -- both storage orders,
    float64 and float32, engines seq / auto / chunked, 1 / 2 / 35 iterations, each layout's strided pass below and above 64
    samples, odd sizes, M == 1, N == 1, batch 1 and 3 and a batch of more than REDUCE_BLOCKS (1184) tiny images; a C-ordered
    batch == the column-major batch of the same images, bit for bit;
  * general inputs: each image within 1e-6 relative of the float64 oracle's DR2L1W_TV, and within 1e-12 of the single-image call;
  * at 4 x 1024^2, in both orders, one solve launches exactly the gather -> chunked -> scatter route for every strided pass (the
    sequential kernel would count as a strided prox launch with no gather and no scatter around it);
  * record / backward: the recorded forward == the no-grad solve bit for bit on every engine; each pass's tape == the batched host
    forward's (test_drw_batched_cpu.forward, dyadic float64); per image gW1, gW2 == proxtv_DR2L1W_TV_vjp_dev_* bit for bit and gY
    within 1e-12 (float64) / 1e-5 (float32); deterministic; NULL weight maps leave gY unchanged;
  * refusals write nothing; torch and numpy surfaces; one 4 x 2048^2 float64 batch against per-image single calls.
"""
import ctypes as C

import numpy as np
import pytest

import dr2_vjp_emu as D
import test_drw_batched_cpu as H
from conftest import relerr
from test_gpu_dr2_vjp import kink_free_difference
from test_gpu_drw_vjp import _p, _st, colmajor, natural, problem
from test_gpu_drw_vjp import record as record1
from test_gpu_drw_vjp import solve as solve1
from test_gpu_drw_vjp import vjp as vjp1

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32


@pytest.fixture
def lib(ptv):
    return ptv.load()


@pytest.fixture
def engine(ptv):
    prev = ptv.set_engine("auto")
    ptv.set_engine(prev)
    yield ptv.set_engine
    ptv.set_engine(prev)


def stack(B, M, N, seed, dt):
    """B dyadic problems (test_gpu_drw_vjp.problem), natural layout: Y (B, M, N), W1 (B, M-1, N), W2 (B, M, N-1)."""
    ps = [problem((M, N), seed + 17 * b, dt) for b in range(B)]
    return tuple(np.stack([p[i] for p in ps]) for i in range(3))


def dev(A, rm, dt):
    return torch.tensor(H.storage(A, rm), dtype=torch.float32 if dt == F32 else torch.float64, device="cuda")


def fn(lib, name, dt):
    return getattr(lib, "proxtv_DR2L1W_TV_batched_%s_%s" % (name, "f32" if dt == F32 else "f64"))


def bsolve(lib, Yd, W1d, W2d, M, N, B, rm, maxit, dt):
    out = torch.full_like(Yd, float("nan"))
    info = np.zeros(3)
    assert fn(lib, "dev", dt)(M, N, B, rm, _p(Yd), _p(W1d), _p(W2d), _p(out), maxit, C.c_void_p(info.ctypes.data), _st()) == 0
    assert info[2] == 0, lib.proxtv_last_error()
    return out


def brecord(lib, Yd, W1d, W2d, M, N, B, rm, maxit, dt, stream=None):
    out = torch.full_like(Yd, float("nan"))
    nb = lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, B, maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    ok = fn(lib, "record_dev", dt)(M, N, B, rm, _p(Yd), _p(W1d), _p(W2d), _p(out), maxit, _p(tape), nb, C.c_void_p(info.ctypes.data),
                                   _st(stream))
    assert ok == 1 and info[2] == 0, lib.proxtv_last_error()
    return out, tape


def bvjp(lib, tape, g, M, N, B, rm, maxit, dt, want1=True, want2=True, stream=None):
    gY = torch.full_like(g, float("nan"))
    gW1 = torch.full((B * (M - 1) * N,), float("nan"), dtype=g.dtype, device="cuda") if want1 else None
    gW2 = torch.full((B * M * (N - 1),), float("nan"), dtype=g.dtype, device="cuda") if want2 else None
    ok = fn(lib, "vjp_dev", dt)(M, N, B, rm, maxit, _p(tape), _p(g), _p(gY), _p(gW1), _p(gW2), _st(stream))
    assert ok == 1, lib.proxtv_last_error()
    return gY, gW1, gW2


def nat(t, B, R, Cc, rm):
    return H.natural(t.cpu().numpy(), B, R, Cc, rm)


def singles(lib, Y, W1, W2, maxit):
    """proxtv_DR2L1W_TV_dev_* on every image (natural layout results)."""
    B, M, N = Y.shape
    return np.stack([natural(solve1(lib, colmajor(Y[b]), colmajor(W1[b]), colmajor(W2[b]), M, N, maxit)) for b in range(B)])


# strided pass of column-major images: rows (length N); of C-ordered images: columns (length M) -- both below and above 64
SHAPES = [(3, 37, 50), (3, 45, 129), (1, 70, 66), (3, 129, 45), (3, 1, 70), (3, 70, 1), (2, 1, 1), (3, 13, 9)]


@pytest.mark.parametrize("maxit", [1, 2, 35])
def test_forward_is_the_single_image_call(lib, engine, maxit):
    it_arg = 0 if maxit == 35 else maxit
    for si, (B, M, N) in enumerate(SHAPES):
        Y64, W1_64, W2_64 = stack(B, M, N, 40 + si, F64)
        for dt in (F64, F32):
            Y, W1, W2 = Y64.astype(dt), W1_64.astype(dt), W2_64.astype(dt)
            for eng in ("seq", "auto", "chunked"):
                engine(eng)
                want = singles(lib, Y, W1, W2, it_arg)
                outs = []
                for rm in (0, 1):
                    what = ((B, M, N), maxit, np.dtype(dt).name, eng, rm)
                    out = bsolve(lib, dev(Y, rm, dt), dev(W1, rm, dt), dev(W2, rm, dt), M, N, B, rm, it_arg, dt)
                    got = nat(out, B, M, N, rm)
                    outs.append(got)
                    assert np.array_equal(got, want), what
                assert np.array_equal(outs[0], outs[1])


def test_forward_more_images_than_reduce_blocks(lib, engine):
    B, M, N = 1300, 3, 5
    Y, W1, W2 = stack(B, M, N, 7, F64)
    for eng in ("auto", "seq"):
        engine(eng)
        want = singles(lib, Y, W1, W2, 2)
        for rm in (0, 1):
            out = bsolve(lib, dev(Y, rm, F64), dev(W1, rm, F64), dev(W2, rm, F64), M, N, B, rm, 2, F64)
            assert np.array_equal(nat(out, B, M, N, rm), want), (eng, rm)


def general(B, M, N, seed):
    """Non-dyadic cfg-like images (blocks plus noise) and positive weights, natural layout."""
    return H.stack((B, M, N), seed, zeros=0.0)


def test_forward_general_inputs_against_oracle(lib, port, engine):
    engine("auto")
    for (B, M, N) in ((3, 96, 130), (2, 130, 40)):
        Y, W1, W2 = general(B, M, N, 5)
        want1 = singles(lib, Y, W1, W2, 0)
        for rm in (0, 1):
            got = nat(bsolve(lib, dev(Y, rm, F64), dev(W1, rm, F64), dev(W2, rm, F64), M, N, B, rm, 0, F64), B, M, N, rm)
            for b in range(B):
                assert relerr(got[b], port.dr2l1w_tv(Y[b], W1[b], W2[b])[0]) <= 1e-6, (B, M, N, rm, b)
                assert relerr(got[b], want1[b]) <= 1e-12, (B, M, N, rm, b)


def read_launches(lib):
    ms, launches, spans = (C.c_double * 3)(), (C.c_longlong * 3)(), (C.c_longlong * 3)()
    lib.proxtv_profile_read(ms, launches, spans)
    return tuple(launches)


def test_no_sequential_route_at_size(lib, engine):
    """(contiguous prox, strided prox, elementwise) launches of one 35-iteration solve (36 pass pairs).  Column-major: W2 gathered once,
    the start value (2), per pair the column prox and gather -> strided prox -> scatter.  C order: W1 gathered once, the start value,
    per pair gather -> strided prox -> scatter of the columns and the row prox -> expand."""
    B, M, N = 4, 1024, 1024
    engine("auto")
    rng = np.random.default_rng(2)
    Y = rng.normal(size=(B, M, N)); W1 = rng.uniform(0.05, 0.5, (B, M - 1, N)); W2 = rng.uniform(0.05, 0.5, (B, M, N - 1))
    for dt in (F32, F64):
        for rm, want in ((0, (36, 36, 1 + 2 + 36 * 2)), (1, (36, 36, 1 + 2 + 36 * 3))):
            args = (dev(Y, rm, dt), dev(W1, rm, dt), dev(W2, rm, dt))
            torch.cuda.synchronize()
            lib.proxtv_profile_reset()
            bsolve(lib, *args, M, N, B, rm, 0, dt)
            assert read_launches(lib) == want, (np.dtype(dt).name, rm, read_launches(lib))


# ---------------------------------------------------------------------------------------------------------------- record / backward
REC_SHAPES = [(3, 37, 50), (2, 45, 129), (3, 129, 45), (3, 1, 70), (3, 70, 1), (2, 1, 1)]


def device_tapes(raw, n, maxit):
    K = 35 if maxit <= 0 else maxit
    nw = D.tape_words(n)
    words = np.asarray(raw)[256:256 + (2 * K + 2) * 2 * nw * 4].view(np.uint32).reshape(2 * K + 2, 2, nw)
    return [(words[p, 0], words[p, 1]) for p in range(2 * K + 2)]


@pytest.mark.parametrize("maxit", [1, 2, 35])
def test_record_tapes_and_backward(lib, engine, port, maxit):
    it_arg = 0 if maxit == 35 else maxit
    for si, (B, M, N) in enumerate(REC_SHAPES):
        Y64, W1_64, W2_64 = stack(B, M, N, 60 + si, F64)
        host = {rm: H.forward(port, Y64, W1_64, W2_64, rm, maxit) for rm in (0, 1)}
        for dt in (F64, F32):
            Y, W1, W2 = Y64.astype(dt), W1_64.astype(dt), W2_64.astype(dt)
            G = np.random.default_rng(si).normal(size=(B, M, N)).astype(dt)
            for eng in ("seq", "auto", "chunked"):
                engine(eng)
                # per image: the single-image record and vjp
                ones = []
                for b in range(B):
                    _, tp = record1(lib, colmajor(Y[b]), colmajor(W1[b]), colmajor(W2[b]), M, N, it_arg)
                    ones.append(vjp1(lib, tp, colmajor(G[b]), M, N, it_arg))
                for rm in (0, 1):
                    what = ((B, M, N), maxit, np.dtype(dt).name, eng, rm)
                    Yd, W1d, W2d = dev(Y, rm, dt), dev(W1, rm, dt), dev(W2, rm, dt)
                    out, tape = brecord(lib, Yd, W1d, W2d, M, N, B, rm, it_arg, dt)
                    assert torch.equal(out, bsolve(lib, Yd, W1d, W2d, M, N, B, rm, it_arg, dt)), what
                    if dt == F64:
                        hout, passes, geo, w = host[rm]
                        assert np.array_equal(out.cpu().numpy(), hout), what
                        for p, (dv, hv) in enumerate(zip(device_tapes(tape.cpu().numpy(), B * M * N, maxit), H.pass_tapes(passes, geo, w))):
                            assert np.array_equal(dv[0], hv[0]) and np.array_equal(dv[1], hv[1]), what + (p,)
                    gY, gW1, gW2 = bvjp(lib, tape, dev(G, rm, dt), M, N, B, rm, it_arg, dt)
                    gY, gW1, gW2 = nat(gY, B, M, N, rm), nat(gW1, B, M - 1, N, rm), nat(gW2, B, M, N - 1, rm)
                    for b, (sY, s1, s2) in enumerate(ones):
                        assert np.array_equal(gW1[b], natural(s1)) and np.array_equal(gW2[b], natural(s2)), what + (b,)
                        assert relerr(gY[b], natural(sY)) <= (1e-12 if dt == F64 else 1e-5), what + (b,)


def test_backward_deterministic_and_null_maps(lib):
    B, M, N = 3, 72, 96
    Y, W1, W2 = stack(B, M, N, 9, F64)
    for rm in (0, 1):
        _, tape = brecord(lib, dev(Y, rm, F64), dev(W1, rm, F64), dev(W2, rm, F64), M, N, B, rm, 5, F64)
        g = torch.randn(B * M * N, dtype=torch.float64, device="cuda")
        a = bvjp(lib, tape, g, M, N, B, rm, 5, F64)
        b = bvjp(lib, tape, g, M, N, B, rm, 5, F64)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        for w1, w2 in ((False, False), (True, False), (False, True)):
            c = bvjp(lib, tape, g, M, N, B, rm, 5, F64, w1, w2)
            assert torch.equal(c[0], a[0]), (rm, w1, w2)
            assert (not w1 or torch.equal(c[1], a[1])) and (not w2 or torch.equal(c[2], a[2]))


def test_refusals_write_nothing(lib):
    B, M, N, K = 2, 40, 70, 3
    Y, W1, W2 = stack(B, M, N, 2, F64)
    rm = 1
    Yd, W1d, W2d = dev(Y, rm, F64), dev(W1, rm, F64), dev(W2, rm, F64)
    _, tape = brecord(lib, Yd, W1d, W2d, M, N, B, rm, K, F64)
    nb = lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, B, K)
    assert nb == 256 + (2 * K + 2) * 2 * (((B * M * N + 31) // 32 * 4 + 255) // 256 * 256)
    assert lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, 0, K) == 0
    assert lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, 1, K) == lib.proxtv_DR2L1W_TV_tape_bytes(M, N, K)
    info = np.zeros(3)
    o = torch.full_like(Yd, 3.0)
    t2 = torch.full((nb,), 7, dtype=torch.uint8, device="cuda")
    rec = lib.proxtv_DR2L1W_TV_batched_record_dev_f64
    bad = ((0, N, B, Yd, W1d, W2d, o, t2, nb), (M, 0, B, Yd, W1d, W2d, o, t2, nb), (M, N, 0, Yd, W1d, W2d, o, t2, nb),
           (M, N, -1, Yd, W1d, W2d, o, t2, nb), (M, N, B, None, W1d, W2d, o, t2, nb), (M, N, B, Yd, None, W2d, o, t2, nb),
           (M, N, B, Yd, W1d, None, o, t2, nb), (M, N, B, Yd, W1d, W2d, None, t2, nb), (M, N, B, Yd, W1d, W2d, o, None, nb),
           (M, N, B, Yd, W1d, W2d, o, t2, nb - 1))
    for i, (m, n, bb, y, w1, w2, out, tp, sz) in enumerate(bad):
        info[:] = 0
        assert rec(m, n, bb, rm, _p(y), _p(w1), _p(w2), _p(out), K, _p(tp), sz, C.c_void_p(info.ctypes.data), None) == 0, i
        assert info[2] == 3, i
    # the forward: negative batch and NULL arrays
    fwd = lib.proxtv_DR2L1W_TV_batched_dev_f64
    for i, (bb, y, w1, w2, out) in enumerate(((-1, Yd, W1d, W2d, o), (B, None, W1d, W2d, o), (B, Yd, None, W2d, o), (B, Yd, W1d, None, o),
                                              (B, Yd, W1d, W2d, None))):
        info[:] = 0
        fwd(M, N, bb, rm, _p(y), _p(w1), _p(w2), _p(out), K, C.c_void_p(info.ctypes.data), None)
        assert info[2] == 3, i
    # vjp: shape, batch, NULL arrays, and every header mismatch -- dtype, shape, batch, order, iterations, a single-image tape, a DR2_TV tape
    g = torch.randn_like(Yd)
    gY = torch.full_like(g, 3.0)
    gW1 = torch.full((B * (M - 1) * N,), 3.0, dtype=torch.float64, device="cuda")
    gW2 = torch.full((B * M * (N - 1),), 3.0, dtype=torch.float64, device="cuda")
    vf = lib.proxtv_DR2L1W_TV_batched_vjp_dev_f64
    for m, n, bb, r, k in ((0, N, B, rm, K), (M, 0, B, rm, K), (M, N, 0, rm, K), (M, N, B, rm, K + 1), (M, N, B, rm, 0), (M + 1, N, B, rm, K),
                           (N, M, B, rm, K), (M, N, B - 1, rm, K), (M, N, B, 1 - rm, K), (M, N, 1, rm, K)):
        assert vf(m, n, bb, r, k, _p(tape), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0, (m, n, bb, r, k)
    assert vf(M, N, B, rm, K, None, _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    assert vf(M, N, B, rm, K, _p(tape), None, _p(gY), _p(gW1), _p(gW2), None) == 0
    assert vf(M, N, B, rm, K, _p(tape), _p(g), None, _p(gW1), _p(gW2), None) == 0
    g32 = g.float(); gY32 = torch.full_like(g32, 3.0)
    assert lib.proxtv_DR2L1W_TV_batched_vjp_dev_f32(M, N, B, rm, K, _p(tape), _p(g32), _p(gY32), None, None, None) == 0
    # a single-image tape given to the batched vjp with batch > 1, and the batched tape given to the single-image vjp
    _, tape1 = record1(lib, colmajor(Y[0]), colmajor(W1[0]), colmajor(W2[0]), M, N, K)
    assert vf(M, N, B, 0, K, _p(tape1), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    assert lib.proxtv_DR2L1W_TV_vjp_dev_f64(M, N, K, _p(tape), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    _, tape0 = brecord(lib, dev(Y, 0, F64), dev(W1, 0, F64), dev(W2, 0, F64), M, N, B, 0, K, F64)
    assert lib.proxtv_DR2L1W_TV_vjp_dev_f64(M, N, K, _p(tape0), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    dr2_tape = torch.zeros(lib.proxtv_DR2_TV_tape_bytes(M, N, B, K), dtype=torch.uint8, device="cuda")
    assert lib.proxtv_DR2_TV_record_dev_f64(M, N, B, rm, _p(Yd), 0.3, 0.3, _p(torch.empty_like(Yd)), K, _p(dr2_tape), dr2_tape.numel(),
                                            None, None) == 1
    assert vf(M, N, B, rm, K, _p(dr2_tape), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    torch.cuda.synchronize()
    assert bool((o == 3.0).all()) and bool((t2 == 7).all())
    assert all(bool((t == 3.0).all()) for t in (gY, gW1, gW2, gY32))


# ---------------------------------------------------------------------------------------------------------------- torch / numpy
def tensors(shape, seed, dt=torch.float64, zeros=0.0):
    B, M, N = shape
    Y, W1, W2 = stack(B, M, N, seed, F64)
    Y = Y + np.random.default_rng(seed).normal(0, 1e-3, Y.shape)             # no ties
    W1[W1 == 0] = 0.05 if zeros == 0.0 else 0.0
    W2[W2 == 0] = 0.05 if zeros == 0.0 else 0.0
    return tuple(torch.tensor(a, dtype=dt, device="cuda") for a in (Y, W1, W2))


def colmajor_images(t):
    """The same (B, H, W) values stored with every image column-major."""
    return t.transpose(1, 2).contiguous().transpose(1, 2)


def test_gradcheck_both_orders(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        for lay in (lambda t: t, colmajor_images):
            x, w1, w2 = (lay(t).requires_grad_(True) for t in tensors((2, 6, 7), 21))
            assert torch.autograd.gradcheck(lambda a, b, c: ptv.tv1w_2d_batched(a, b, c, max_iters=3), (x, w1, w2), eps=1e-6, atol=1e-6)
        x, w1, w2 = (t.requires_grad_(True) for t in tensors((2, 5, 70), 22))        # the chunked contiguous row pass of C order
        assert torch.autograd.gradcheck(lambda a, b, c: ptv.tv1w_2d_batched(a, b, c, max_iters=2), (x, w1, w2), eps=1e-6, atol=1e-6)


def test_directional_differences(ptv):
    for shape, lay in (((2, 96, 130), lambda t: t), ((2, 130, 40), colmajor_images)):
        Y, W1, W2 = (lay(t) for t in tensors(shape, 8))
        G = torch.randn(shape, dtype=torch.float64, device="cuda")
        f = lambda a, b, c: ptv.tv1w_2d_batched(a, b, c, max_iters=5)           # noqa: E731
        x, w1, w2 = (t.clone().requires_grad_(True) for t in (Y, W1, W2))
        (f(x, w1, w2) * G).sum().backward()
        with torch.no_grad():
            base = f(Y, W1, W2)
            for i, grad in enumerate((x.grad, w1.grad, w2.grad)):
                V = torch.randn_like(grad)

                def step(e):
                    args = [Y, W1, W2]
                    args[i] = args[i] + e * V
                    return ((f(*args) - base) * G).sum().item()
                fd = kink_free_difference(step)
                an = (grad * V).sum().item()
                assert abs(fd - an) <= 2e-6 * max(abs(an), 1.0), (shape, i, fd, an)


def test_forward_equals_no_grad_and_each_input_alone(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            for lay in (lambda t: t, colmajor_images):
                Y, W1, W2 = (lay(t) for t in tensors((3, 50, 90), 4, dt, zeros=0.2))
                G = torch.randn(Y.shape, dtype=dt, device="cuda")
                ref = ptv.tv1w_2d_batched(Y, W1, W2)
                assert ref.grad_fn is None and ref.stride() == Y.stride()
                with torch.no_grad():
                    assert ptv.tv1w_2d_batched(Y.clone().requires_grad_(True), W1, W2).grad_fn is None
                full = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
                out = ptv.tv1w_2d_batched(*full)
                assert out.grad_fn is not None and torch.equal(out.detach(), ref), (eng, dt)
                out.backward(G)
                for i in range(3):
                    args = [Y, W1, W2]
                    args[i] = args[i].clone().requires_grad_(True)
                    o = ptv.tv1w_2d_batched(*args)
                    assert torch.equal(o.detach(), ref)
                    o.backward(G)
                    assert torch.equal(args[i].grad, full[i].grad), (eng, dt, i)
            # on dyadic data each image is tv1w_2d on that image, forward and weight gradients bit for bit
            for lay in (lambda t: t, colmajor_images):
                Yd, W1d, W2d = (lay(torch.tensor(a, dtype=dt, device="cuda")) for a in stack(3, 40, 70, 31, F64))
                G = torch.randn(Yd.shape, dtype=dt, device="cuda")
                full = [t.clone().requires_grad_(True) for t in (Yd, W1d, W2d)]
                out = ptv.tv1w_2d_batched(*full)
                out.backward(G)
                for b in range(3):
                    one = [t[b].clone().requires_grad_(True) for t in (Yd, W1d, W2d)]
                    o = ptv.tv1w_2d(*one)
                    assert torch.equal(o.detach(), out.detach()[b]), (eng, dt, b)
                    o.backward(G[b])
                    assert torch.equal(one[1].grad, full[1].grad[b]) and torch.equal(one[2].grad, full[2].grad[b]), (eng, dt, b)
                    assert relerr(one[0].grad.cpu().numpy(), full[0].grad[b].cpu().numpy()) <= (1e-12 if dt == torch.float64 else 1e-5)


def test_expanded_mixed_dtypes_views_and_streams(ptv):
    B, M, N = 3, 48, 80
    Y, W1, W2 = tensors((B, M, N), 6)
    G = torch.randn((B, M, N), dtype=torch.float64, device="cuda")
    # float32 images, float64 weights: the weight gradients come back in float64, equal to the float32 call's
    x = Y.float().requires_grad_(True)
    w1, w2 = W1.clone().requires_grad_(True), W2.clone().requires_grad_(True)
    ptv.tv1w_2d_batched(x, w1, w2).backward(G.float())
    x32, a32, b32 = (t.float().requires_grad_(True) for t in (Y, W1, W2))
    ptv.tv1w_2d_batched(x32, a32, b32).backward(G.float())
    assert w1.grad.dtype == torch.float64 and torch.equal(w1.grad, a32.grad.double()) and torch.equal(w2.grad, b32.grad.double())
    assert torch.equal(x.grad, x32.grad)
    # one weight map for every image through expand (and a learned scalar): autograd sums the per-image gradients
    for lay in (lambda t: t, colmajor_images):
        m1 = W1[0].clone().requires_grad_(True)
        s2 = torch.tensor(0.4, dtype=torch.float64, device="cuda", requires_grad=True)
        ptv.tv1w_2d_batched(lay(Y), m1.expand(B, M - 1, N), s2.expand(B, M, N - 1)).backward(lay(G))
        f1 = W1[0].expand(B, M - 1, N).clone().requires_grad_(True)
        f2 = torch.full((B, M, N - 1), 0.4, dtype=torch.float64, device="cuda", requires_grad=True)
        ptv.tv1w_2d_batched(lay(Y), f1, f2).backward(lay(G))
        assert relerr(m1.grad.cpu().numpy(), f1.grad.sum(0).cpu().numpy()) <= 1e-12
        assert abs(s2.grad.item() - f2.grad.sum().item()) <= 1e-12 * max(abs(f2.grad).sum().item(), 1.0)
    # views: a slice and a permuted tensor are made contiguous and give the contiguous input's gradient
    xc = Y.clone().requires_grad_(True)
    ptv.tv1w_2d_batched(xc, W1, W2).backward(G)
    for make in (lambda: torch.nn.functional.pad(Y, (0, 3))[:, :, :N], lambda: Y.permute(1, 0, 2).contiguous().permute(1, 0, 2)):
        leaf = make().detach().requires_grad_(True)
        out = ptv.tv1w_2d_batched(leaf, W1, W2)
        assert torch.equal(out.detach(), ptv.tv1w_2d_batched(Y, W1, W2))
        out.backward(G)
        assert torch.equal(leaf.grad, xc.grad)
    # a non-default stream
    a = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
    ptv.tv1w_2d_batched(*a).backward(G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
        ptv.tv1w_2d_batched(*b).backward(G)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, q.grad) for p, q in zip(a, b))


def test_numpy_equals_torch(ptv):
    B, M, N = 3, 45, 70
    Y, W1, W2 = general(B, M, N, 12)
    for dt, tdt in ((F64, torch.float64), (F32, torch.float32)):
        got = ptv.tv1w_2d_batched(Y.astype(dt), W1, W2, max_iters=7)
        assert got.dtype == dt and got.flags.c_contiguous and got.shape == (B, M, N)
        want = ptv.tv1w_2d_batched(*(torch.tensor(a, dtype=tdt, device="cuda") for a in (Y.astype(dt), W1, W2)), max_iters=7)
        assert np.array_equal(got, want.cpu().numpy()), np.dtype(dt).name
        # a Fortran-ordered array is the same values
        assert np.array_equal(ptv.tv1w_2d_batched(np.asfortranarray(Y.astype(dt)), W1, W2, max_iters=7), got)


def test_at_size_2048(lib):
    """Dyadic float64 inputs (exact per-image sums): the batch's forward and weight gradients equal the single calls' bit for bit."""
    B, M, N = 4, 2048, 2048
    rng = np.random.default_rng(4)
    Y = np.round((np.repeat(np.repeat(rng.normal(0, 1, (B, M // 16, N // 16)), 16, axis=1), 16, axis=2) + rng.normal(0, 0.3, (B, M, N))) * 256) / 256
    W1 = np.round(rng.uniform(0.05, 0.5, (B, M - 1, N)) * 256) / 256
    W2 = np.round(rng.uniform(0.05, 0.5, (B, M, N - 1)) * 256) / 256
    G = rng.normal(size=(B, M, N))
    rm = 1
    Yd, W1d, W2d = dev(Y, rm, F64), dev(W1, rm, F64), dev(W2, rm, F64)
    out, tape = brecord(lib, Yd, W1d, W2d, M, N, B, rm, 0, F64)
    gY, gW1, gW2 = bvjp(lib, tape, dev(G, rm, F64), M, N, B, rm, 0, F64)
    del tape
    out, gY, gW1, gW2 = nat(out, B, M, N, rm), nat(gY, B, M, N, rm), nat(gW1, B, M - 1, N, rm), nat(gW2, B, M, N - 1, rm)
    for b in range(B):
        y1, w1, w2 = colmajor(Y[b]), colmajor(W1[b]), colmajor(W2[b])
        o1, t1 = record1(lib, y1, w1, w2, M, N, 0)
        assert np.array_equal(out[b], natural(o1)), b
        sY, s1, s2 = vjp1(lib, t1, colmajor(G[b]), M, N, 0)
        del t1
        assert np.array_equal(gW1[b], natural(s1)) and np.array_equal(gW2[b], natural(s2)), b
        assert relerr(gY[b], natural(sY)) <= 1e-12, b
