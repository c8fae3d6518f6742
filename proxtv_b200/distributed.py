"""Multi-GPU driver for the one case the path shards: a BATCH of independent images (BASELINE config 5).

One process per GPU (torchrun); rank `src` holds the batch, every rank solves a contiguous slab of images with the
single-GPU path (`proxtv_b200.tv1_2d_batched`), and the slabs are gathered back on `src`.  There is no communication
inside a solve: a single image cannot be split without an all-to-all transpose between the two passes of every
iteration (SURVEY.md 8e), which the north star excludes.  Collectives: one scatter and one gather of image slabs
(point-to-point sends grouped with `batch_isend_irecv`, so uneven slabs need no padding) over NCCL/NVLink, or gloo on CPU
for the host-logic tests.
"""
import numpy as np


def slab_bounds(batch, world):
    """Contiguous, balanced split of `batch` images over `world` ranks: returns [(start, stop)] per rank."""
    base, extra = divmod(int(batch), int(world))
    out, s = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append((s, s + n))
        s += n
    return out


def _peer(group, r):
    """Global rank of group member r (P2POp peers and broadcast sources are global ranks)."""
    import torch.distributed as dist
    return r if group is None else dist.get_global_rank(group, r)


def tv1_2d_batched_sharded(x, w, max_iters=0, src=0, group=None, solver=None, device=None, pieces=1, timings=None):
    """DR2_TV on every image of x (B, H, W), sharded over the ranks of `group`.

    x       on rank `src` (a rank index inside `group`): torch tensor or numpy array (float32 / float64); ignored elsewhere
    solver  callable(local (b, H, W) tensor, w, max_iters) -> tensor; default: the CUDA path of this package
    pieces  > 1: every rank's slab is cut into that many pieces and the transfers are pipelined with the solves -- piece k + 1
            is received (and the result of piece k - 1 sent back) while piece k is being solved, so that only the first
            piece's scatter and the last piece's gather are exposed
    timings optional dict: receives the wall time of the phases on this rank ('scatter', 'solve', 'gather' seconds; with
            pieces > 1 the phases overlap and only 'total' is meaningful)
    Returns the (B, H, W) result on rank `src`, None on the other ranks.
    """
    import time
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group); world = dist.get_world_size(group)
    backend = dist.get_backend(group)
    if pieces > 1:
        return _sharded_pipelined(x, w, max_iters, src, group, solver, device, pieces, timings)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    meta = [None]
    if rank == src:
        xt = torch.as_tensor(x)
        assert xt.dim() == 3 and xt.dtype in (torch.float32, torch.float64)
        meta = [(tuple(xt.shape), str(xt.dtype).split(".")[-1])]
    dist.broadcast_object_list(meta, src=_peer(group, src), group=group)
    (B, H, W), dname = meta[0]
    dtype = getattr(torch, dname)
    bounds = slab_bounds(B, world)
    lo, hi = bounds[rank]
    local = torch.empty((hi - lo, H, W), dtype=dtype, device=device)

    # ---- scatter ----
    ops = []
    if rank == src:
        xs = xt.to(device).contiguous()
        for r, (a, b) in enumerate(bounds):
            if r == src:
                local.copy_(xs[a:b])
            elif b > a:
                ops.append(dist.P2POp(dist.isend, xs[a:b].contiguous(), _peer(group, r), group))
    elif hi > lo:
        ops.append(dist.P2POp(dist.irecv, local, _peer(group, src), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()

    # ---- local solve (no communication) ----
    if solver is None:
        from . import tv1_2d_batched
        solver = lambda t, ww, it: tv1_2d_batched(t, ww, max_iters=it)      # noqa: E731
    res = solver(local, w, max_iters) if hi > lo else local
    res = torch.as_tensor(res).to(device=device, dtype=dtype).contiguous()

    # ---- gather ----
    ops = []; out = None
    if rank == src:
        out = torch.empty((B, H, W), dtype=dtype, device=device)
        for r, (a, b) in enumerate(bounds):
            if r == src:
                out[a:b].copy_(res)
            elif b > a:
                ops.append(dist.P2POp(dist.irecv, out[a:b], _peer(group, r), group))
    elif hi > lo:
        ops.append(dist.P2POp(dist.isend, res, _peer(group, src), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return out


def _sharded_pipelined(x, w, max_iters, src, group, solver, device, pieces, timings):
    """Software-pipelined variant: transfers of neighbouring pieces overlap the solve of the current one."""
    import time
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group); world = dist.get_world_size(group)
    backend = dist.get_backend(group)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    meta = [None]
    if rank == src:
        xt = torch.as_tensor(x)
        assert xt.dim() == 3 and xt.dtype in (torch.float32, torch.float64)
        meta = [(tuple(xt.shape), str(xt.dtype).split(".")[-1])]
    dist.broadcast_object_list(meta, src=_peer(group, src), group=group)
    (B, H, W), dname = meta[0]
    dtype = getattr(torch, dname)
    bounds = slab_bounds(B, world)
    if solver is None:
        from . import tv1_2d_batched
        solver = lambda t, ww, it: tv1_2d_batched(t, ww, max_iters=it)      # noqa: E731
    # piece p of rank r: images [a + cut(p), a + cut(p + 1)) of its slab [a, b)
    def cut(a, b, p):
        return a + (b - a) * p // pieces
    sync = (lambda: torch.cuda.synchronize()) if device.type == "cuda" else (lambda: None)
    t0 = time.perf_counter()
    xs = xt.to(device).contiguous() if rank == src else None
    out = torch.empty((B, H, W), dtype=dtype, device=device) if rank == src else None
    lo, hi = bounds[rank]
    bufs = [None] * pieces; res = [None] * pieces
    pending = []

    def post_scatter(p):
        ops = []
        if rank == src:
            for r, (a, b) in enumerate(bounds):
                pa, pb = cut(a, b, p), cut(a, b, p + 1)
                if r == src:
                    bufs[p] = xs[pa:pb]
                elif pb > pa:
                    ops.append(dist.P2POp(dist.isend, xs[pa:pb], _peer(group, r), group))
        else:
            pa, pb = cut(lo, hi, p), cut(lo, hi, p + 1)
            bufs[p] = torch.empty((pb - pa, H, W), dtype=dtype, device=device)
            if pb > pa:
                ops.append(dist.P2POp(dist.irecv, bufs[p], _peer(group, src), group))
        return dist.batch_isend_irecv(ops) if ops else []

    def post_gather(p):
        ops = []
        if rank == src:
            for r, (a, b) in enumerate(bounds):
                pa, pb = cut(a, b, p), cut(a, b, p + 1)
                if r == src:
                    out[pa:pb].copy_(res[p])
                elif pb > pa:
                    ops.append(dist.P2POp(dist.irecv, out[pa:pb], _peer(group, r), group))
        elif res[p].shape[0] > 0:
            ops.append(dist.P2POp(dist.isend, res[p], _peer(group, src), group))
        return dist.batch_isend_irecv(ops) if ops else []

    reqs = {0: post_scatter(0)}
    for p in range(pieces):
        for q in reqs.pop(p):
            q.wait()
        if p + 1 < pieces:
            reqs[p + 1] = post_scatter(p + 1)                # next piece travels while this one is solved
        r_ = solver(bufs[p], w, max_iters) if bufs[p].shape[0] > 0 else bufs[p]
        res[p] = torch.as_tensor(r_).to(device=device, dtype=dtype).contiguous()
        sync()                                               # the result must be complete before it is sent
        pending.append(post_gather(p))
        bufs[p] = None
    for g in pending:
        for q in g:
            q.wait()
    sync()
    if timings is not None:
        timings["total"] = time.perf_counter() - t0
    return out


# ======================================================================================================================
# ONE image over several GPUs (SURVEY.md 8f N3)
# ======================================================================================================================
def _lane_passes():
    """The two passes of a Douglas-Rachford iteration on this rank's slabs, as launches of the lane engine through the C ABI
    (proxtv_lane_prox_dev_*: device pointers, current stream).  Slabs are column-major, held as row-major tensors [columns][rows]."""
    import torch
    from . import _dev_call, require_device
    require_device()                               # refuse here, before the first exchange, rather than inside the iteration

    def cols(t_c, w):                              # t_c [n_cols][M]: every column is a contiguous fiber
        out = torch.empty_like(t_c)
        _dev_call("lane_prox_dev", t_c, 0, t_c, None, None, out, t_c.shape[0], t_c.shape[1], 1, float(w))
        return out

    def rows(final, y_r, x1_r, t_r, w):            # slabs [N][m]: row fibers have stride m, adjacent rows are adjacent in memory
        out = torch.empty_like(t_r)
        _dev_call("lane_prox_dev", t_r, 2 if final else 1, y_r, x1_r, t_r, out, t_r.shape[1], t_r.shape[0], t_r.shape[1], float(w))
        return out

    return cols, rows


def tv1_2d_single_sharded(x, w, max_iters=0, src=0, group=None, passes=None, device=None, timings=None):
    """DR2_TV of ONE image (M x N) split over the ranks of `group`: the only way a single large image scales past one GPU.

    The fibers of one pass are independent, but the two passes of an iteration need orthogonal partitions: rank r owns the column
    block r for the column pass and the row block r for the row pass, and the iterate changes partition twice per iteration with an
    all-to-all (each rank keeps 1/G of its slab and exchanges the rest: (G-1)/G of the array crosses NVLink per exchange).  The
    arithmetic is the single-GPU staged schedule's (solver.cu: dr2_lane_body): x1 = prox_cols(t); t' = (t - x1) + prox_rows(Y -
    (2 (t - x1) - t)); only the summation order of the start value 2 * mean differs (per-rank partial sums), i.e. rounding level.

    x        on rank `src`: (M, N) numpy array or torch tensor (float64 / float32); ignored elsewhere.  M and N must be multiples of
             the group size (and the slabs must suit the lane engine: even slab widths).
    passes   optional (prox_cols(t_c, w), row_pass(final, y_r, x1_r, t_r, w)) callables on slabs [columns][rows]; default: the lane
             engine on this rank's GPU.  The CPU tests pass oracle-backed stand-ins and run this driver over gloo.
    timings  optional dict: 'exchange' = seconds this rank spent in the all-to-alls (and their pack / unpack copies), 'total'.
    Returns the (M, N) result on rank `src` (numpy in -> numpy out), None on the other ranks.
    """
    import time
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group); G = dist.get_world_size(group)
    backend = dist.get_backend(group)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    sync = (lambda: torch.cuda.synchronize(device)) if device.type == "cuda" else (lambda: None)
    t_start = time.perf_counter(); t_x = [0.0]
    meta = [None]; was_numpy = False
    if rank == src:
        was_numpy = isinstance(x, np.ndarray)
        xt = torch.as_tensor(x)
        assert xt.dim() == 2 and xt.dtype in (torch.float32, torch.float64)
        meta = [(tuple(xt.shape), str(xt.dtype).split(".")[-1])]
    dist.broadcast_object_list(meta, src=_peer(group, src), group=group)
    (M, N), dname = meta[0]
    dtype = getattr(torch, dname)
    if M % G or N % G:
        raise ValueError("tv1_2d_single_sharded: both image dimensions must be multiples of the group size (%d x %d over %d ranks)" % (M, N, G))
    m, n = M // G, N // G
    maxit = int(max_iters) if max_iters and max_iters > 0 else 35              # src/TV2Dopt.cpp:387
    if passes is None:
        passes = _lane_passes()
    prox_cols, row_pass = passes

    def all_to_all(send):                          # [G][n][m] -> [G][n][m], chunk g goes to / comes from rank g
        recv = torch.empty_like(send)
        if timings is None:                        # no host synchronisation on the fast path: NCCL orders itself against the stream
            dist.all_to_all_single(recv, send, group=group)
            return recv
        sync(); t0 = time.perf_counter()
        dist.all_to_all_single(recv, send, group=group)
        sync(); t_x[0] += time.perf_counter() - t0
        return recv

    def cols_to_rows(a_c):                         # column slab [n][M] -> row slab [N][m]
        return all_to_all(a_c.view(n, G, m).permute(1, 0, 2).contiguous()).view(N, m)

    def rows_to_cols(a_r):                         # row slab [N][m] -> column slab [n][M]
        return all_to_all(a_r.view(G, n, m)).permute(1, 0, 2).contiguous().view(n, M)

    # ---- distribute: column slabs of Y (column-major image == tensor [N][M]); the row slabs follow by the same exchange ----
    y_c = torch.empty((n, M), dtype=dtype, device=device)
    if rank == src:
        full = xt.to(device).t().contiguous()                                   # [N][M]
        chunks = list(full.view(G, n, M).unbind(0))
    ops = []
    if rank == src:
        for r in range(G):
            if r == src:
                y_c.copy_(chunks[r])
            else:
                ops.append(dist.P2POp(dist.isend, chunks[r].contiguous(), _peer(group, r), group))
    else:
        ops.append(dist.P2POp(dist.irecv, y_c, _peer(group, src), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    y_r = cols_to_rows(y_c)
    # ---- start value 2 * mean (:390-395) ----
    s = y_c.sum(dtype=torch.float64).reshape(1)
    dist.all_reduce(s, group=group)
    t0v = (2.0 * s / float(M * N)).to(dtype)
    t_c = t0v.expand(n, M).contiguous(); t_r = t0v.expand(N, m).contiguous()
    out_r = None
    for it in range(maxit + 1):
        final = it == maxit
        x1_c = t_c if (it == 0 and maxit > 0) else prox_cols(t_c, w)           # the prox of the constant start image is that constant
        x1_r = cols_to_rows(x1_c) if not (it == 0 and maxit > 0) else t_r
        if final:
            out_r = row_pass(True, y_r, x1_r, t_r, w)
        else:
            t_r = row_pass(False, y_r, x1_r, t_r, w)
            t_c = rows_to_cols(t_r)
    # ---- collect the row slabs on src: out[N][M], slab r = columns of rows r*m .. (r+1)*m ----
    res = None; ops = []
    if rank == src:
        parts = [torch.empty((N, m), dtype=dtype, device=device) for _ in range(G)]
        for r in range(G):
            if r == src:
                parts[r].copy_(out_r)
            else:
                ops.append(dist.P2POp(dist.irecv, parts[r], _peer(group, r), group))
    else:
        ops.append(dist.P2POp(dist.isend, out_r.contiguous(), _peer(group, src), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    sync()
    if rank == src:
        res = torch.cat(parts, dim=1).t()                                       # [N][M] column-major -> (M, N) view
        if was_numpy:
            res = res.cpu().numpy()
    if timings is not None:
        timings["exchange"] = t_x[0]; timings["total"] = time.perf_counter() - t_start
    return res
