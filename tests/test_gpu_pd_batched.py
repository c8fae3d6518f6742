"""GPU tests (-m gpu) of the batched proximal Dykstra solvers (DESIGN.md section 16): proxtv_PD*_TV_batched_* and tvgen_batched.

Bars:
  * forward: under seq and chunked every item's x and info row == the single-item proxtv_PD*_TV_dev_* on that item into a fresh
    buffer, bit for bit -- float64 and float32, PD_TV with 1, 3 and 5 terms (one axis repeated), PD2_TV with 1 and 2 terms, 1D to 3D
    items, B in {1, 3, 7}, odd item sizes (slots that are not 16-byte aligned), and items that stop at different K (a constant item,
    smooth items, noisy items the cap ends); under auto and lane to 1e-12 relative with equal K;
  * the recorded forward == the no-grad batched call bit for bit, and the tape's K table == info[:, 0];
  * backward under seq and chunked: every item's gY == the single-item vjp for that item bit for bit, glam within 1e-12 of the
    single-item glam (times npen for PD_TV: the batched glam is of the penalties as given), a NULL glam leaves gY unchanged;
  * refusals write nothing: the single-item tapes, the other solver's batched tape, a wrong batch or maxIters, a short tape;
  * tvgen_batched: a batch of one == torch tvgen bit for bit, gradcheck on a batch that mixes items ended by the cap with items ended
    by the stop rule (every item's K asserted at every evaluation), forward with grad == without, C order / item-column-major /
    non-contiguous view, ws as list / ndarray / tensor never modified, the ws gradient, a non-default stream, numpy == numpy tvgen.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _a(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _st(stream=None):
    return C.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def sfx(dt):
    return "f32" if dt in (np.float32, torch.float32) else "f64"


def tdt(dt):
    return torch.float32 if dt == np.float32 else torch.float64


def name(pd2):
    return "PD2_TV" if pd2 else "PD_TV"


@pytest.fixture
def lib(ptv):
    return ptv.load()


@pytest.fixture
def engine(ptv):
    prev = ptv.set_engine("auto")
    ptv.set_engine(prev)
    yield ptv.set_engine
    ptv.set_engine(prev)


def item(kind, ns, seed):
    """One column-major item, flat: 'const', 'smooth' (stops well below 1000 iterations) or 'noisy' (runs to a small cap)."""
    n = int(np.prod(ns))
    if kind == "const":
        return np.full(n, 0.7)
    if kind == "smooth":
        g = np.meshgrid(*[np.arange(k) for k in ns], indexing="ij")
        return sum(np.sin(c / (5.0 + a) + seed) for a, c in enumerate(g)).ravel(order="F")
    return np.random.default_rng(seed).normal(size=n)


KINDS = ["noisy", "const", "smooth", "noisy", "smooth", "const", "noisy"]


def batch_input(ns, B, seed, dt):
    return np.concatenate([item(KINDS[b % len(KINDS)], ns, seed + b) for b in range(B)]).astype(dt)


def single(lib, pd2, y, ns, ws, ds, maxit):
    """proxtv_PD*_TV_dev_* on one flat item tensor, into a fresh buffer."""
    lam, dsa, nsa = np.array(ws, dtype=np.float64), np.array(ds, dtype=np.float64), np.array(ns, dtype=np.int32)   # alive for the call
    out = torch.full_like(y, float("nan"))
    info = np.zeros(3)
    f = getattr(lib, "proxtv_%s_dev_%s" % (name(pd2), sfx(y.dtype)))
    assert f(_p(y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _st()) == 1, lib.proxtv_last_error()
    return out, info


def single_record(lib, pd2, y, ns, ws, ds, maxit):
    nsa = np.array(ns, dtype=np.int32)
    nb = getattr(lib, "proxtv_%s_tape_bytes" % name(pd2))(_a(nsa), len(ns), len(ws), maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    out = torch.full_like(y, float("nan"))
    info = np.zeros(3)
    lam, dsa = np.array(ws, dtype=np.float64), np.array(ds, dtype=np.float64)
    f = getattr(lib, "proxtv_%s_record_dev_%s" % (name(pd2), sfx(y.dtype)))
    assert f(_p(y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _p(tape), nb, _st()) == 1, lib.proxtv_last_error()
    return out, info, tape


def single_vjp(lib, pd2, tape, g, ns, ds, maxit, K):
    gY = torch.full_like(g, float("nan"))
    glam = torch.full((len(ds),), float("nan"), dtype=torch.float64, device="cuda")
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    f = getattr(lib, "proxtv_%s_vjp_dev_%s" % (name(pd2), sfx(g.dtype)))
    assert f(_a(nsa), len(ns), len(ds), _a(dsa), maxit, K, _p(tape), _p(g), _p(gY), _p(glam), _st()) == 1, lib.proxtv_last_error()
    return gY, glam


def tape_bytes(lib, pd2, ns, npen, B, maxit):
    nsa = np.array(ns, dtype=np.int32)
    return getattr(lib, "proxtv_%s_batched_tape_bytes" % name(pd2))(_a(nsa), len(ns), npen, B, maxit)


def batched(lib, pd2, Y, ns, ws, ds, B, maxit, record=False, stream=None):
    """proxtv_PD*_TV_batched_dev_* (or _record_dev_*) on the flat tensor Y of B items; returns (out, info (B, 3), tape or None)."""
    lam = np.array(ws, dtype=np.float64)
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    out = torch.full_like(Y, float("nan"))
    info = np.zeros(3 * B)
    args = [_p(Y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), B, maxit]
    tape = None
    if record:
        nb = tape_bytes(lib, pd2, ns, len(ws), B, maxit)
        tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        args += [_p(tape), nb]
    f = getattr(lib, "proxtv_%s_batched_%sdev_%s" % (name(pd2), "record_" if record else "", sfx(Y.dtype)))
    assert f(*args, _st(stream)) == 1, lib.proxtv_last_error()
    assert np.array_equal(lam, np.array(ws, dtype=np.float64))          # never written
    return out, info.reshape(B, 3), tape


def batched_vjp(lib, pd2, tape, G, ns, ds, B, maxit, want_glam=True):
    gY = torch.full_like(G, float("nan"))
    glam = torch.full((B * len(ds),), float("nan"), dtype=torch.float64, device="cuda") if want_glam else None
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    f = getattr(lib, "proxtv_%s_batched_vjp_dev_%s" % (name(pd2), sfx(G.dtype)))
    rc = f(_a(nsa), len(ns), len(ds), _a(dsa), B, maxit, _p(tape), _p(G), _p(gY), _p(glam), _st())
    assert rc == 1, lib.proxtv_last_error()
    return gY, glam


# (pd2, ns, ws, ds): PD_TV with 1, 3, 5 terms (one axis repeated), PD2_TV with 1 and 2 terms; 1D to 3D; odd sizes misalign the slots
CASES = [(False, (301,), [0.4], [1]),
         (False, (12, 10, 8), [0.2, 0.25, 0.3], [1, 2, 3]),
         (False, (11, 9, 5), [0.2, 0.25, 0.3], [1, 2, 3]),
         (False, (9, 8, 7), [0.1, 0.2, 0.15, 0.1, 0.05], [1, 2, 3, 1, 2]),
         (True, (33, 17), [0.3], [2]),
         (True, (40, 36), [0.3, 0.2], [1, 2]),
         (True, (13, 11, 7), [0.2, 0.3], [3, 1])]
IDS = ["pd-1d-odd", "pd-3d", "pd-3d-odd", "pd-5terms", "pd2-1term-odd", "pd2-2d", "pd2-3d-odd"]


def check_items(lib, pd2, Y, out, info, ns, ws, ds, B, maxit, exact, what):
    n = int(np.prod(ns))
    for b in range(B):
        ref, rinfo = single(lib, pd2, Y[b * n:(b + 1) * n].clone(), ns, ws, ds, maxit)
        got = out[b * n:(b + 1) * n]
        if exact:
            assert torch.equal(got, ref) and np.array_equal(info[b], rinfo), (what, b, info[b], rinfo)
        else:
            assert info[b, 0] == rinfo[0], (what, b, info[b], rinfo)
            err = (got.double() - ref.double()).abs().max().item() / max(ref.double().abs().max().item(), 1e-300)
            assert err <= (1e-12 if Y.dtype == torch.float64 else 1e-5), (what, b, err)


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("maxit", [4, 0])
def test_forward_equals_single_items(lib, engine, case, maxit):
    pd2, ns, ws, ds = case
    for dt in (np.float64, np.float32):
        for B in (1, 3, 7):
            Y = torch.tensor(batch_input(ns, B, 5, dt), device="cuda")
            for eng in ("seq", "chunked"):
                engine(eng)
                out, info, _ = batched(lib, pd2, Y, ns, ws, ds, B, maxit)
                check_items(lib, pd2, Y, out, info, ns, ws, ds, B, maxit, True, (name(pd2), ns, B, eng, np.dtype(dt).name))
            if B == 7 and maxit == 0 and len(ws) > 1:                        # one term: every item stops at K = 2 (PD_TV) or 1 (PD2_TV)
                assert len(set(info[:, 0].tolist())) >= 2, info                # the items stop at different K


@pytest.mark.parametrize("case", [CASES[1], CASES[5]], ids=["pd-3d", "pd2-2d"])
def test_forward_stop_rule_under_a_large_cap(lib, engine, case):
    """maxIters = 1000: smooth items stop on their own test, the constant one at once, the noisy ones run on; still bit for bit."""
    pd2, ns, ws, ds = case
    for dt in (np.float64, np.float32):
        Y = torch.tensor(np.concatenate([item(k, ns, 9) for k in ("smooth", "const", "smooth")]).astype(dt), device="cuda")
        engine("chunked")
        out, info, _ = batched(lib, pd2, Y, ns, ws, ds, 3, 1000)
        assert np.all(info[:, 0] < 1000) and np.all(info[:, 1] <= 1e-6), info
        check_items(lib, pd2, Y, out, info, ns, ws, ds, 3, 1000, True, (name(pd2), np.dtype(dt).name))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_forward_auto_and_lane(lib, engine, case):
    pd2, ns, ws, ds = case
    for dt in (np.float64,):
        Y = torch.tensor(batch_input(ns, 7, 5, dt), device="cuda")
        for eng in ("auto", "lane"):
            engine(eng)
            out, info, _ = batched(lib, pd2, Y, ns, ws, ds, 7, 4)
            check_items(lib, pd2, Y, out, info, ns, ws, ds, 7, 4, False, (name(pd2), ns, eng))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_recorded_forward_and_backward(lib, engine, case):
    pd2, ns, ws, ds = case
    n = int(np.prod(ns))
    B = 7
    for dt in (np.float64, np.float32):
        Y = torch.tensor(batch_input(ns, B, 8, dt), device="cuda")
        G = torch.tensor(np.random.default_rng(4).normal(size=B * n).astype(dt), device="cuda")
        for eng in ("seq", "chunked"):
            engine(eng)
            what = (name(pd2), ns, eng, np.dtype(dt).name)
            out, info, tape = batched(lib, pd2, Y, ns, ws, ds, B, 0, record=True)
            ref, rinfo, _ = batched(lib, pd2, Y, ns, ws, ds, B, 0)
            assert torch.equal(out, ref) and np.array_equal(info, rinfo), what
            assert np.array_equal(tape[256:256 + 4 * B].cpu().numpy().view(np.int32), info[:, 0].astype(np.int32)), what
            gY, glam = batched_vjp(lib, pd2, tape, G, ns, ds, B, 0)
            gY2, _ = batched_vjp(lib, pd2, tape, G, ns, ds, B, 0, want_glam=False)
            assert torch.equal(gY, gY2), what
            glam = glam.cpu().numpy().reshape(B, len(ds))
            for b in range(B):
                _, sinfo, stape = single_record(lib, pd2, Y[b * n:(b + 1) * n].clone(), ns, ws, ds, 0)
                K = int(sinfo[0])
                assert K == int(info[b, 0]), what
                sY, slam = single_vjp(lib, pd2, stape, G[b * n:(b + 1) * n].clone(), ns, ds, 0, K)
                assert torch.equal(gY[b * n:(b + 1) * n], sY), (what, b)
                want = slam.cpu().numpy() * (1.0 if pd2 else float(len(ds)))
                assert np.abs(glam[b] - want).max() <= 1e-12 * max(np.abs(want).max(), 1e-300), (what, b, glam[b], want)


def test_refusals_write_nothing(lib):
    ns, ws, ds, B = (12, 10), [0.2, 0.3, 0.1], [1, 2, 1], 3
    n = int(np.prod(ns))
    Y = torch.tensor(batch_input(ns, B, 3, np.float64), device="cuda")
    _, _, tape = batched(lib, False, Y, ns, ws, ds, B, 5, record=True)
    _, _, tape2 = batched(lib, True, Y, ns, ws[:2], ds[:2], B, 5, record=True)
    _, _, stape = single_record(lib, False, Y[:n].clone(), ns, ws, ds, 5)
    G = torch.ones(B * n, dtype=torch.float64, device="cuda")
    vf = lib.proxtv_PD_TV_batched_vjp_dev_f64
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)

    def refused(tp, batch=B, maxit=5):
        gY = torch.full_like(G, float("nan"))
        glam = torch.full((B * 3,), float("nan"), dtype=torch.float64, device="cuda")
        assert vf(_a(nsa), 2, 3, _a(dsa), batch, maxit, _p(tp), _p(G), _p(gY), _p(glam), _st()) == 0
        assert torch.isnan(gY).all() and torch.isnan(glam).all()
        return lib.proxtv_last_error().decode()
    assert "not a batched PD_TV tape" in refused(stape)
    assert "not a batched PD_TV tape" in refused(tape2)
    assert "another batch" in refused(tape, batch=2)
    assert "maxIters" in refused(tape, maxit=6)
    # the single-item vjp refuses the batched tape
    gY = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
    assert lib.proxtv_PD_TV_vjp_dev_f64(_a(nsa), 2, 3, _a(dsa), 5, 5, _p(tape), _p(G), _p(gY), None, _st()) == 0
    assert torch.isnan(gY).all()
    # a short tape, and batch < 1: nothing written but the RC of every item
    lam = np.array(ws, dtype=np.float64)
    out = torch.full_like(Y, float("nan"))
    info = np.full(3 * B, -5.0)
    nb = tape_bytes(lib, False, ns, 3, B, 5)
    short = torch.zeros(nb - 1, dtype=torch.uint8, device="cuda")
    rf = lib.proxtv_PD_TV_batched_record_dev_f64
    assert rf(_p(Y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), 2, 3, B, 5, _p(short), nb - 1, _st()) == 0
    assert torch.isnan(out).all() and np.array_equal(info.reshape(B, 3)[:, :2], np.full((B, 2), -5.0)) and np.all(info[2::3] == 3)
    assert (short == 0).all() and np.array_equal(lam, np.array(ws))
    assert lib.proxtv_PD_TV_batched_dev_f64(_p(Y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), 2, 3, 0, 5, _st()) == 0
    assert torch.isnan(out).all()


# ---------------------------------------------------------------------------------------------------------------- tvgen_batched
def test_batch_of_one_equals_tvgen(ptv, engine):
    for eng in ("auto", "chunked"):
        engine(eng)
        for ws, ds in (([0.2, 0.3, 0.25], [1, 2, 3]), ([0.3, 0.2], [1, 3])):
            x = torch.tensor(np.random.default_rng(1).normal(size=(10, 9, 8)), device="cuda")
            want = ptv.tvgen(x, ws, ds, [1] * len(ws))
            winfo = ptv.tvgen.last_info.copy()
            got = ptv.tvgen_batched(x[None], ws, ds, [1] * len(ws))
            assert torch.equal(got[0], want) and np.array_equal(ptv.tvgen_batched.last_info[0], winfo)


def test_layouts_and_ws_untouched(ptv, engine):
    engine("chunked")
    rng = np.random.default_rng(2)
    base = torch.tensor(rng.normal(size=(4, 9, 7, 5)), device="cuda")
    base[1] = 0.5                                                   # an item that stops early
    wl = [0.2, 0.3, 0.25]
    wn = np.array(wl)
    wt = torch.tensor(wl, dtype=torch.float64, device="cuda")
    fcol = base.permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)   # items column-major, batch slowest
    assert not fcol.is_contiguous()
    view = torch.tensor(rng.normal(size=(4, 9, 14, 5)), device="cuda")[:, :, ::2]
    for x in (base, fcol, view):
        for w in (wl, wn, wt):
            got = ptv.tvgen_batched(x, w, [1, 2, 3], [1, 1, 1])
            info = ptv.tvgen_batched.last_info.copy()
            assert got.shape == x.shape and (got.stride() == x.stride() or x is view)
            for b in range(4):
                xb = x[b] if x is not view else x[b].contiguous()
                want = ptv.tvgen(xb, wl, [1, 2, 3], [1, 1, 1])
                assert torch.equal(got[b], want) and np.array_equal(info[b], ptv.tvgen.last_info), b
            if x is base:
                assert len(set(info[:, 0].tolist())) == 2, info                # the constant item stops first
        assert wl == [0.2, 0.3, 0.25] and np.array_equal(wn, [0.2, 0.3, 0.25])
        assert torch.equal(wt, torch.tensor([0.2, 0.3, 0.25], dtype=torch.float64, device="cuda"))


def capped_items(ptv, f, K):
    def g(*a):
        y = f(*a)
        assert np.array_equal(ptv.tvgen_batched.last_info[:, 0], K), ptv.tvgen_batched.last_info
        return y
    return g


def test_gradcheck(ptv, engine):
    """Items 0 and 2 run to the cap (3), item 1 is constant and stops on its own test: PD_TV at K = 2 (it starts from x = 0), PD2_TV
    at K = 1 (it starts from x = y)."""
    for eng in ("seq", "chunked"):
        engine(eng)
        x = torch.tensor(np.random.default_rng(3).normal(size=(3, 5, 4, 3)), device="cuda")
        x[1] = 0.4
        x.requires_grad_(True)
        w = torch.tensor([0.2, 0.3, 0.25], dtype=torch.float64, device="cuda", requires_grad=True)
        f = capped_items(ptv, lambda a, b: ptv.tvgen_batched(a, b, [1, 2, 3], [1, 1, 1], max_iters=3), [3, 2, 3])
        assert torch.autograd.gradcheck(f, (x, w), eps=1e-6, atol=1e-6)
        x2 = torch.tensor(np.random.default_rng(4).normal(size=(3, 6, 5)), device="cuda")
        x2[1] = 0.4
        x2.requires_grad_(True)
        w2 = torch.tensor([0.3, 0.2], dtype=torch.float64, device="cuda", requires_grad=True)
        f2 = capped_items(ptv, lambda a, b: ptv.tvgen_batched(a, b, [1, 2], [1, 1], max_iters=3), [3, 1, 3])
        assert torch.autograd.gradcheck(f2, (x2, w2), eps=1e-6, atol=1e-6)


def test_forward_with_grad_and_ws_gradient(ptv, engine):
    engine("chunked")
    x = torch.tensor(batch_input((8, 7, 6), 5, 2, np.float32).reshape(5, 6, 7, 8), device="cuda")
    w = torch.tensor([0.2, 0.3, 0.25], dtype=torch.float32, device="cuda", requires_grad=True)
    xr = x.clone().requires_grad_(True)
    y = ptv.tvgen_batched(xr, w, [1, 2, 3], [1, 1, 1])
    assert torch.equal(y, ptv.tvgen_batched(x, w.detach(), [1, 2, 3], [1, 1, 1]))
    G = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (xr, w), G)
    want_gw = torch.zeros(3, dtype=torch.float64, device="cuda")
    for b in range(5):
        xb = x[b].clone().requires_grad_(True)
        wb = w.detach().clone().requires_grad_(True)
        yb = ptv.tvgen(xb, wb, [1, 2, 3], [1, 1, 1])
        assert torch.equal(yb, y[b])
        gxb, gwb = torch.autograd.grad(yb, (xb, wb), G[b])
        assert torch.equal(gxb, gx[b])
        want_gw += gwb.double()
    assert torch.allclose(gw.double(), want_gw, rtol=1e-5, atol=0)


def test_non_default_stream(ptv, engine):
    engine("chunked")
    x = torch.tensor(batch_input((20, 16), 3, 6, np.float64).reshape(3, 16, 20), device="cuda")
    want = ptv.tvgen_batched(x, [0.3, 0.2], [1, 2], [1, 1])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = ptv.tvgen_batched(x, [0.3, 0.2], [1, 2], [1, 1])
    s.synchronize()
    assert torch.equal(got, want)


def test_numpy_equals_numpy_tvgen(ptv, engine):
    engine("chunked")
    x = batch_input((9, 8, 7), 4, 1, np.float64).reshape(4, 7, 8, 9)
    for ws, ds in (([0.2, 0.3, 0.25], [1, 2, 3]), ([0.3, 0.2], [2, 3]), ([0.4], [3])):
        got = ptv.tvgen_batched(x, ws, ds, [1] * len(ws))
        info = ptv.tvgen_batched.last_info.copy()
        assert got.shape == x.shape and got.dtype == np.float64
        for b in range(4):
            assert np.array_equal(got[b], ptv.tvgen(x[b], list(ws), ds, [1] * len(ws))), (ws, b)
            assert np.array_equal(info[b], ptv.tvgen.last_info), (ws, b)
    g32 = ptv.tvgen_batched(x.astype(np.float32), [0.3, 0.2], [1, 2], [1, 1])
    assert g32.dtype == np.float32
