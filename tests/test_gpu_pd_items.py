"""GPU tests (-m gpu) of per-item penalties for the batched proximal Dykstra solvers (DESIGN.md section 16.1):
proxtv_PD*_TV_batched_items_*, the per-fiber prox and tape entries, and tvgen_batched with a (B, npen) ws.

Bars:
  * per-fiber prox: fiber j of proxtv_prox_fibers_lamf_dev_* == the uniform pass with lamf[j / fpi] (np.array_equal) on its engine:
    seq, chunked, and lane for a positive table (whole fibers, and forced chunking with every boundary repaired; warps that straddle
    two groups), a table with a zero going to the chunked kernels under lane and auto, auto with a positive table within 1e-12 of
    chunked; float64 and float32, contiguous and strided fibers, long and short fibers, fpi 1, 7, 32, 33, penalties 0 and 1e-12 .. 1e4;
    its tape == the uniform tape per fiber, and a tape whose groups are not whole slabs is refused;
  * per-item forward under seq and chunked: every item's x and info row == proxtv_PD*_TV_dev_* on that item with its own row, bit for
    bit, over the section 16 cases (PD_TV 1, 3, 5 terms; PD2_TV 1, 2; 1D..3D; B 1, 3, 7; odd sizes; items stopping at different K),
    with an item whose penalties are zero; under auto and lane to 1e-12 relative (float32: 1e-5) with equal K;
  * equal rows == the shared-row _batched_ call, result and info bit for bit, on every engine;
  * recorded forward == no-grad forward; the batched vjp of its tape gives each item's gY bit for bit and glam within 1e-12 of the
    single-item vjp with that item's row;
  * tvgen_batched: gradcheck with a (B, npen) ws, an expanded ws gets the summed gradient, layouts, a non-default stream, ws never
    modified, numpy == a numpy loop of tvgen(x[b], ws[b]).
"""
import numpy as np
import pytest

from test_gpu_pd_batched import (CASES, IDS, _a, _p, _st, batch_input, batched, batched_vjp, capped_items, engine, lib,  # noqa: F401
                                 name, sfx, single, single_record, single_vjp, tape_bytes)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

VALUES = [0.0, 1e-12, 1e-6, 0.01, 0.3, 1.0, 100.0, 1e4]


def fibers(a, nf, L, inc):
    """(nf, L) view of the fibers (nf, L, inc) of a flat array: fiber j at (j / inc) inc L + j % inc, stride inc."""
    return a.reshape(nf // inc, L, inc).transpose(0, 2, 1).reshape(nf, L)


def uniform(lib, y, nf, L, inc, lam):
    out = torch.full_like(y, float("nan"))
    f = getattr(lib, "proxtv_prox_fibers_dev_%s" % sfx(y.dtype))
    assert f(_p(y), _p(out), nf, L, inc, lam, None, _st()) == 1, lib.proxtv_last_error()
    return out


def tape_bits(lib, y, nf, L, inc, lam=None, lamf=None, fpi=1):
    nw = ((nf * L + 31) // 32 * 4 + 255) // 256 * 64
    F = torch.zeros(nw, dtype=torch.int32, device="cuda"); U = torch.zeros_like(F)
    if lamf is None:
        rc = getattr(lib, "proxtv_fiber_tape_dev_%s" % sfx(y.dtype))(_p(y), nf, L, inc, lam, None, _p(F), _p(U), _st())
    else:
        rc = getattr(lib, "proxtv_fiber_tape_lamf_dev_%s" % sfx(y.dtype))(_p(y), nf, L, inc, _p(lamf), fpi, _p(F), _p(U), _st())
    assert rc == 1, lib.proxtv_last_error()
    bits = lambda t: np.unpackbits(t.cpu().numpy().view(np.uint8), bitorder="little")[:nf * L]   # noqa: E731
    return bits(F), bits(U)


def per_fiber(lib, y, nf, L, inc, lamf, fpi):
    out = torch.full_like(y, float("nan"))
    f = getattr(lib, "proxtv_prox_fibers_lamf_dev_%s" % sfx(y.dtype))
    assert f(_p(y), _p(out), nf, L, inc, _p(lamf), fpi, _st()) == 1, lib.proxtv_last_error()
    return out


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("fpi", [1, 7, 32, 33])
@pytest.mark.parametrize("L", [96, 40])
@pytest.mark.parametrize("inc", [1, 8], ids=["contig", "strided"])
def test_per_fiber_prox_equals_uniform_pass(ptv, lib, engine, dt, fpi, L, inc):
    """Enough fibers (>= 1024) for the lane route.  A table with a zero entry: seq and chunked bit for bit their uniform passes, lane and
    auto the chunked one (a zero keeps the table off the lane engine).  A positive table: lane bit for bit the uniform lane pass of each
    penalty -- also with forced chunking and every chunk boundary repaired (halo 0) -- and auto within 1e-12 (float32: 1e-5) of chunked."""
    grp = fpi * 8 // np.gcd(fpi, 8)                       # a multiple of fpi and of the strided layout's 8 fibers per slab
    nf = grp * (-(-1024 // grp))
    rng = np.random.default_rng(fpi * 100 + L + inc)
    y = torch.tensor((rng.normal(size=nf * L) * 3.0).astype(dt), device="cuda")
    groups = nf // fpi
    of = np.arange(nf) // fpi
    tables = {"zero": np.array([VALUES[(g * 3) % len(VALUES)] for g in range(groups)]),
              "positive": np.array([VALUES[1 + (g * 3) % (len(VALUES) - 1)] for g in range(groups)])}
    for kind, vals in tables.items():
        lamf = torch.tensor(vals.astype(dt), device="cuda")
        for eng, tuning in (("seq", None), ("chunked", None), ("lane", None), ("lane", (32, 0)), ("auto", None)):
            if kind == "zero" and tuning:
                continue
            engine(eng)
            if tuning:
                ptv.load().proxtv_lane_tuning(tuning[0], tuning[1], -1)
            try:
                got = fibers(per_fiber(lib, y, nf, L, inc, lamf, fpi).cpu().numpy(), nf, L, inc)
                exact = eng in ("seq", "chunked") or (eng == "lane" and kind == "positive") or (eng == "auto" and kind == "zero")
                ref_eng = eng if eng in ("seq", "chunked") or (eng == "lane" and kind == "positive") else "chunked"
                engine(ref_eng)
                for v in np.unique(vals):
                    sel = vals[of] == v
                    want = fibers(uniform(lib, y, nf, L, inc, float(dt(v))).cpu().numpy(), nf, L, inc)
                    if exact:
                        assert np.array_equal(got[sel], want[sel]), (kind, eng, tuning, v)
                    else:
                        err = np.abs(got[sel].astype(np.float64) - want[sel]).max() / max(np.abs(want[sel]).max(), 1e-300)
                        assert err <= (1e-12 if dt == np.float64 else 1e-5), (kind, eng, v, err)
            finally:
                if tuning:
                    ptv.load().proxtv_lane_tuning(0, 32, -1)
        engine("seq")
        out = per_fiber(lib, y, nf, L, inc, lamf, fpi)
        if fpi % inc == 0:
            F, U = tape_bits(lib, out, nf, L, inc, lamf=lamf, fpi=fpi)
            idx = fibers(np.arange(nf * L), nf, L, inc)
            for v in np.unique(vals):
                Fu, Uu = tape_bits(lib, out, nf, L, inc, lam=float(dt(v)))
                e = idx[vals[of] == v].ravel()
                assert np.array_equal(F[e], Fu[e]) and np.array_equal(U[e], Uu[e]), v
        else:                                             # a group that is not whole slabs is refused
            F = torch.full((64,), 7, dtype=torch.int32, device="cuda")
            assert getattr(lib, "proxtv_fiber_tape_lamf_dev_%s" % sfx(dt))(_p(out), nf, L, inc, _p(lamf), fpi, _p(F), _p(F), _st()) == 0
            torch.cuda.synchronize()
            assert torch.all(F == 7)


def test_per_fiber_prox_refusals(lib):
    y = torch.zeros(64, dtype=torch.float64, device="cuda")
    out = torch.full_like(y, 5.0)
    tab = torch.full((4,), 0.1, dtype=torch.float64, device="cuda")
    f = lib.proxtv_prox_fibers_lamf_dev_f64
    for args in ((8, 8, 1, _p(tab), 0), (8, 8, 1, _p(tab), 3), (8, 8, 1, None, 2), (8, 8, 0, _p(tab), 2)):
        assert f(_p(y), _p(out), *args, _st()) == 0
    F = torch.full((64,), 7, dtype=torch.int32, device="cuda")
    t = lib.proxtv_fiber_tape_lamf_dev_f64
    for args in ((8, 8, 1, _p(tab), 0), (8, 8, 1, _p(tab), 3), (8, 8, 1, None, 2), (8, 8, 2, _p(tab), 1)):
        assert t(_p(y), *args, _p(F), _p(F), _st()) == 0
    torch.cuda.synchronize()
    assert torch.all(out == 5.0) and torch.all(F == 7)


def rows(B, npen, seed, zero_item=1):
    W = np.random.default_rng(seed).uniform(0.1, 0.5, size=(B, npen))
    if B > zero_item:
        W[zero_item] = 0.0
    return W


def items_call(lib, pd2, Y, ns, W, ds, B, maxit, record=False, stream=None):
    """proxtv_PD*_TV_batched_items_dev_* (or _items_record_dev_*); returns (out, info (B, 3), tape or None)."""
    lam = np.ascontiguousarray(W, dtype=np.float64).ravel()
    keep = lam.copy()
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    out = torch.full_like(Y, float("nan"))
    info = np.zeros(3 * B)
    args = [_p(Y), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ds), B, maxit]
    tape = None
    if record:
        nb = tape_bytes(lib, pd2, ns, len(ds), B, maxit)
        tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        args += [_p(tape), nb]
    f = getattr(lib, "proxtv_%s_batched_items_%sdev_%s" % (name(pd2), "record_" if record else "", sfx(Y.dtype)))
    assert f(*args, _st(stream)) == 1, lib.proxtv_last_error()
    assert np.array_equal(lam, keep)                                    # never written
    return out, info.reshape(B, 3), tape


def check_items_rows(lib, pd2, Y, out, info, ns, W, ds, B, maxit, exact, what):
    n = int(np.prod(ns))
    for b in range(B):
        ref, rinfo = single(lib, pd2, Y[b * n:(b + 1) * n].clone(), ns, list(W[b]), ds, maxit)
        got = out[b * n:(b + 1) * n]
        if exact:
            assert torch.equal(got, ref) and np.array_equal(info[b], rinfo), (what, b, info[b], rinfo)
        else:
            assert info[b, 0] == rinfo[0], (what, b, info[b], rinfo)
            err = (got.double() - ref.double()).abs().max().item() / max(ref.double().abs().max().item(), 1e-300)
            assert err <= (1e-12 if Y.dtype == torch.float64 else 1e-5), (what, b, err)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_items_forward_equals_single_items(lib, engine, case):
    pd2, ns, ws, ds = case
    for dt in (np.float64, np.float32):
        for B in (1, 3, 7):
            Y = torch.tensor(batch_input(ns, B, 5, dt), device="cuda")
            W = rows(B, len(ds), B)
            for eng in ("seq", "chunked"):
                engine(eng)
                out, info, _ = items_call(lib, pd2, Y, ns, W, ds, B, 0)
                check_items_rows(lib, pd2, Y, out, info, ns, W, ds, B, 0, True, (name(pd2), ns, eng, B, np.dtype(dt).name))
        Y = torch.tensor(batch_input(ns, 7, 5, dt), device="cuda")
        W = rows(7, len(ds), 9)
        for eng in ("auto", "lane"):
            engine(eng)
            out, info, _ = items_call(lib, pd2, Y, ns, W, ds, 7, 4)
            check_items_rows(lib, pd2, Y, out, info, ns, W, ds, 7, 4, False, (name(pd2), ns, eng))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_equal_rows_equal_shared_call(lib, engine, case):
    pd2, ns, ws, ds = case
    B = 7
    Y = torch.tensor(batch_input(ns, B, 6, np.float64), device="cuda")
    W = np.tile(np.array(ws, dtype=np.float64), (B, 1))
    for eng in ("seq", "chunked", "lane", "auto"):
        engine(eng)
        out, info, _ = items_call(lib, pd2, Y, ns, W, ds, B, 0)
        ref, rinfo, _ = batched(lib, pd2, Y, ns, ws, ds, B, 0)
        assert torch.equal(out, ref) and np.array_equal(info, rinfo), (name(pd2), ns, eng)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_items_recorded_forward_and_backward(lib, engine, case):
    pd2, ns, ws, ds = case
    n = int(np.prod(ns))
    B = 7
    W = rows(B, len(ds), 11)
    for dt in (np.float64, np.float32):
        Y = torch.tensor(batch_input(ns, B, 8, dt), device="cuda")
        G = torch.tensor(np.random.default_rng(4).normal(size=B * n).astype(dt), device="cuda")
        for eng in ("seq", "chunked"):
            engine(eng)
            what = (name(pd2), ns, eng, np.dtype(dt).name)
            out, info, tape = items_call(lib, pd2, Y, ns, W, ds, B, 0, record=True)
            ref, rinfo, _ = items_call(lib, pd2, Y, ns, W, ds, B, 0)
            assert torch.equal(out, ref) and np.array_equal(info, rinfo), what
            gY, glam = batched_vjp(lib, pd2, tape, G, ns, ds, B, 0)
            glam = glam.cpu().numpy().reshape(B, len(ds))
            for b in range(B):
                _, sinfo, stape = single_record(lib, pd2, Y[b * n:(b + 1) * n].clone(), ns, list(W[b]), ds, 0)
                K = int(sinfo[0])
                assert K == int(info[b, 0]), what
                sY, slam = single_vjp(lib, pd2, stape, G[b * n:(b + 1) * n].clone(), ns, ds, 0, K)
                assert torch.equal(gY[b * n:(b + 1) * n], sY), (what, b)
                want = slam.cpu().numpy() * (1.0 if pd2 else float(len(ds)))
                assert np.abs(glam[b] - want).max() <= 1e-12 * max(np.abs(want).max(), 1e-300), (what, b, glam[b], want)


def test_gradcheck_per_item_ws(ptv, engine):
    """Items 0 and 2 run to the cap (3), item 1 is constant and stops on its own test (PD_TV at K = 2, PD2_TV at K = 1)."""
    for eng in ("seq", "chunked"):
        engine(eng)
        x = torch.tensor(np.random.default_rng(3).normal(size=(3, 5, 4, 3)), device="cuda")
        x[1] = 0.4
        x.requires_grad_(True)
        w = torch.tensor([[0.2, 0.3, 0.25], [0.1, 0.15, 0.05], [0.35, 0.2, 0.3]], dtype=torch.float64, device="cuda", requires_grad=True)
        f = capped_items(ptv, lambda a, b: ptv.tvgen_batched(a, b, [1, 2, 3], [1, 1, 1], max_iters=3), [3, 2, 3])
        assert torch.autograd.gradcheck(f, (x, w), eps=1e-6, atol=1e-6)
        x2 = torch.tensor(np.random.default_rng(4).normal(size=(3, 6, 5)), device="cuda")
        x2[1] = 0.4
        x2.requires_grad_(True)
        w2 = torch.tensor([[0.3, 0.2], [0.25, 0.1], [0.15, 0.35]], dtype=torch.float64, device="cuda", requires_grad=True)
        f2 = capped_items(ptv, lambda a, b: ptv.tvgen_batched(a, b, [1, 2], [1, 1], max_iters=3), [3, 1, 3])
        assert torch.autograd.gradcheck(f2, (x2, w2), eps=1e-6, atol=1e-6)


def test_per_item_gradient_rows_and_expanded_ws(ptv, engine):
    engine("chunked")
    x = torch.tensor(batch_input((8, 7, 6), 5, 2, np.float64).reshape(5, 6, 7, 8), device="cuda")
    W = torch.tensor(rows(5, 3, 12), dtype=torch.float32, device="cuda", requires_grad=True)
    y = ptv.tvgen_batched(x, W, [1, 2, 3], [1, 1, 1])
    G = torch.randn_like(y)
    (gW,) = torch.autograd.grad(y, (W,), G)
    xr = x.clone().requires_grad_(True)                              # x alone requiring grad: no ws gradient is formed
    (gx,) = torch.autograd.grad(ptv.tvgen_batched(xr, W.detach(), [1, 2, 3], [1, 1, 1]), (xr,), G)
    assert torch.isfinite(gx).all()
    assert gW.shape == (5, 3) and gW.dtype == torch.float32
    for b in range(5):
        wb = W.detach()[b].double().clone().requires_grad_(True)
        yb = ptv.tvgen(x[b], wb, [1, 2, 3], [1, 1, 1])
        assert torch.equal(yb, y[b])
        (gwb,) = torch.autograd.grad(yb, (wb,), G[b])
        assert torch.allclose(gW[b].double(), gwb, rtol=1e-5, atol=1e-7), b
    # an expanded shared ws: each item sees the same row, autograd sums the rows into w's gradient
    w = torch.tensor([0.2, 0.3, 0.25], dtype=torch.float64, device="cuda", requires_grad=True)
    ye = ptv.tvgen_batched(x, w.expand(5, 3), [1, 2, 3], [1, 1, 1])
    w1 = w.detach().clone().requires_grad_(True)
    ys = ptv.tvgen_batched(x, w1, [1, 2, 3], [1, 1, 1])
    assert torch.equal(ye, ys)
    (ge,) = torch.autograd.grad(ye, (w,), G)
    (gs,) = torch.autograd.grad(ys, (w1,), G)
    assert torch.allclose(ge, gs, rtol=1e-12, atol=0)


def test_layouts_stream_and_ws_untouched(ptv, engine):
    engine("chunked")
    rng = np.random.default_rng(2)
    base = torch.tensor(rng.normal(size=(4, 9, 7, 5)), device="cuda")
    base[1] = 0.5
    Wl = [[0.2, 0.3, 0.25], [0.0, 0.1, 0.2], [0.4, 0.05, 0.3], [0.15, 0.15, 0.15]]
    Wn = np.array(Wl)
    Wt = torch.tensor(Wl, dtype=torch.float32, device="cuda")
    fcol = base.permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)   # items column-major, batch slowest
    for x in (base, fcol):
        for W in (Wl, Wn, Wt):
            got = ptv.tvgen_batched(x, W, [1, 2, 3], [1, 1, 1])
            info = ptv.tvgen_batched.last_info.copy()
            assert got.shape == x.shape and got.stride() == x.stride()
            for b in range(4):
                wb = [float(v) for v in np.asarray(Wn[b], dtype=np.float32 if W is Wt else np.float64)]
                want = ptv.tvgen(x[b], wb, [1, 2, 3], [1, 1, 1])
                assert torch.equal(got[b], want) and np.array_equal(info[b], ptv.tvgen.last_info), b
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            got2 = ptv.tvgen_batched(x, Wn, [1, 2, 3], [1, 1, 1])
        s.synchronize()
        assert torch.equal(got2, ptv.tvgen_batched(x, Wn, [1, 2, 3], [1, 1, 1]))
    assert Wl[1] == [0.0, 0.1, 0.2] and np.array_equal(Wn, np.array(Wl))
    assert torch.equal(Wt, torch.tensor(Wl, dtype=torch.float32, device="cuda"))


def test_numpy_equals_numpy_tvgen_loop(ptv, engine):
    engine("chunked")
    x = batch_input((9, 8, 7), 4, 1, np.float64).reshape(4, 7, 8, 9)
    for ds in ([1, 2, 3], [2, 3], [3]):
        W = rows(4, len(ds), 5)
        got = ptv.tvgen_batched(x, W, ds, [1] * len(ds))
        info = ptv.tvgen_batched.last_info.copy()
        assert got.shape == x.shape and got.dtype == np.float64
        for b in range(4):
            assert np.array_equal(got[b], ptv.tvgen(x[b], list(W[b]), ds, [1] * len(ds))), (ds, b)
            assert np.array_equal(info[b], ptv.tvgen.last_info), (ds, b)
    g32 = ptv.tvgen_batched(x.astype(np.float32), rows(4, 2, 6), [1, 2], [1, 1])
    assert g32.dtype == np.float32
