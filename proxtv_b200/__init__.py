"""proxtv_b200 -- H100-native (sm_90a) Total-Variation (TV-L1) proximity operators behind proxTV's Python surface.

Drop-in for the hot path of ``prox_tv`` (reference: prox_tv/__init__.py): ``tv1_1d`` (:124), ``tv1w_1d`` (:218),
``tv1_2d`` (:355) and ``tvgen`` (:533) keep the reference's names, argument meaning, dtype/layout coercion, assertion
behaviour and return conventions; the computation runs in hand-written sm_90a CUDA kernels reached through the C ABI of
``libproxtv_b200.so`` (include/proxtv_b200.h).  There is NO CPU fallback: without the built extension or a CUDA
device the calls raise.

Extensions the reference lacks (SURVEY.md section 8b): a leading batch dimension (``tv1_1d_batched``,
``tv1w_1d_batched``, ``tv1_2d_batched``, ``tv1w_2d_batched``), float32, and torch CUDA tensors as inputs (device-resident path: no PCIe
traffic, no host transposes -- a C-ordered tensor is handled by swapping the kernels' stride roles).  The batched 1D functions,
``tv1_2d`` ('dr' and 'pd') / ``tv1_2d_batched`` ('dr'), ``tv1w_2d`` / ``tv1w_2d_batched`` ('dr') and the N-D ``tvgen`` / ``tvgen_pdr`` are differentiable on torch
tensors (exact backward kernels); the converged 2D solvers ('condat', 'chambolle-pock') are too with ``backward='converged'``, through
the Jacobian of the prox at the partition the forward reached.

Every call into the library goes through ``_host_call`` (numpy: host arrays) or ``_dev_call`` (torch: device pointers on the tensor's
current stream), which share one failure rule (``_check``).  Each 2D family has one numpy body (``_tv2_numpy``, ``_tv2w_numpy``) on the
``proxtv_*_batched_*`` host symbols, a single image being a column-major batch of one; the taped 2D solvers share one autograd Function
(``TV2``) and one table of what differs between them (``_TAPED``); the N-D solvers share one front (``_tvgen_front``), one tensor layout
(``_nd_layout``) and one Function (``ND``).
"""
import ctypes as C
import functools
import types

import numpy as np

from . import _lib
from ._lib import ProxTVError, load, require_device  # noqa: F401

__all__ = ["tv1_1d", "tv1w_1d", "tv1_2d", "tv1w_2d", "tvgen", "tvgen_pdr", "tv1_1d_batched", "tv1w_1d_batched", "tv1_2d_batched",
           "tv1w_2d_batched", "tvgen_batched", "set_engine", "set_pinned_results", "ProxTVError"]

_N_INFO = 3                      # prox_tv/__init__.py:67
ENGINES = {"auto": 0, "seq": 1, "chunked": 2, "chunked-strided": 3, "pipelined": 4, "tspace": 5, "tpose": 6, "lane": 7, "lane-t": 8}


def set_engine(name):
    """Select the kernel family / DR schedule ('auto' | 'seq' | 'chunked' | 'chunked-strided' | 'pipelined' | 'tspace' |
    'tpose' | 'lane' | 'lane-t', see include/proxtv_b200.h); returns the previous one.  Only measurements and tests need this."""
    prev = load().proxtv_set_engine(ENGINES[name])
    return [k for k, v in ENGINES.items() if v == prev][0]


# ---- argument coercion, as the reference does it (prox_tv/__init__.py:80-121) ----
def force_float_scalar(x):
    return x if isinstance(x, float) else float(x)


def force_float_matrix(x):
    if not isinstance(x, np.ndarray):
        try:
            x = np.array(x)
        except Exception:
            raise TypeError("Input must be a numpy matrix or compatible object")
    if x.dtype != np.dtype("float64"):
        return x.astype("float")
    return x


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def _is_torch(x):
    return type(x).__module__.startswith("torch") and hasattr(x, "data_ptr")


def _check(ok, name, rc=True, info=None):
    """The one failure rule of the entry points: a zero return where the entry returns 1 on success (rc), or RC = 3 in any row of the
    info array the call filled.  Raises ProxTVError naming the C symbol."""
    if (rc and not ok) or (info is not None and np.any(info[2::_N_INFO] == 3)):
        raise ProxTVError("%s failed: %s" % (name, _lib.last_error()))


def _host_call(entry, ref, *args, rc=True, info=None):
    """Call proxtv_<entry>_f32 / _f64 (by the numpy array ref's dtype), or with ref None the symbol named entry as it is; ndarrays in
    args go as host pointers, None as NULL.  Raises ProxTVError naming the symbol when the call fails (_check)."""
    name = entry if ref is None else "proxtv_%s_%s" % (entry, "f32" if ref.dtype == np.float32 else "f64")
    fn = getattr(require_device(), name)
    _check(fn(*[_ptr(a) if isinstance(a, np.ndarray) else a for a in args]), name, rc, info)


# ---- torch CUDA tensors: device calls and autograd ----
def _dev_call(entry, ref, *args, rc=True, info=None):
    """Call proxtv_<entry>_f32 / _f64 (by ref's dtype) on ref's device, with ref's current CUDA stream appended to args; torch
    tensors in args go as device pointers, numpy arrays as host pointers, None as NULL.  Raises ProxTVError naming the entry point
    when the call fails (_check)."""
    import torch
    name = "proxtv_%s_%s" % (entry, "f32" if ref.dtype == torch.float32 else "f64")
    fn = getattr(require_device(), name)
    args = [C.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else _ptr(a) if isinstance(a, np.ndarray) else a for a in args]
    with torch.cuda.device(ref.device):
        ok = fn(*args, C.c_void_p(torch.cuda.current_stream(ref.device).cuda_stream))
    _check(ok, name, rc, info)


def _needs_grad(*objs):
    """Grad mode is on and one of objs is a torch tensor that requires grad: the solve must be recorded for a backward."""
    import torch
    return torch.is_grad_enabled() and any(_is_torch(t) and t.requires_grad for t in objs)


def _w_float(w):
    """(the penalty w as a float, w when it is a tensor else None); the solve takes the float, the tensor only receives the gradient."""
    w_t = w if _is_torch(w) else None
    return (float(w_t.detach()) if w_t is not None else float(w)), w_t


def _penalty_grad(g, like):
    """The gradient of a penalty tensor, like = its (dtype, device, shape), from g, the gradients of the penalties the solve used:
    summed in float64 for a 0-dim tensor (one penalty for all of them), then cast to the tensor's dtype and device."""
    import torch
    dtype, device, shape = like
    if len(shape) == 0:
        g = g.sum(dtype=torch.float64)
    return g.to(dtype=dtype, device=device).reshape(shape)


# ---- result arrays in pooled page-locked memory ----
# The reference returns a fresh ``np.zeros`` array.  For a 128 MiB image that costs more than the solve: 32768 page faults when the
# device-to-host copy first touches the pages, and a pageable copy at a fraction of the PCIe rate.  Large results are therefore
# carved out of a small pool of page-locked blocks (cudaHostAlloc through the library); a block returns to the pool when the last
# array that refers to it -- the result or any view of it -- is garbage-collected.  ``set_pinned_results(False)`` switches it off.
class _PinnedPool:
    MIN_BYTES = 1 << 20          # smaller results: plain numpy memory
    MAX_IDLE = 1 << 30           # idle blocks kept for reuse (bytes)

    def __init__(self):
        self.enabled = True
        self.free = []           # (capacity, address)

    def empty(self, shape, dtype, order):
        import weakref
        dtype = np.dtype(dtype)
        nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
        if not self.enabled or nbytes < self.MIN_BYTES:
            return np.zeros(shape, dtype=dtype, order=order)
        lib = load()
        fit = [b for b in self.free if nbytes <= b[0] <= 2 * nbytes]
        if fit:
            blk = min(fit); self.free.remove(blk)
        else:
            addr = lib.proxtv_host_alloc(nbytes)
            if not addr:
                return np.zeros(shape, dtype=dtype, order=order)
            blk = (nbytes, addr)
        buf = (C.c_char * nbytes).from_address(blk[1])
        weakref.finalize(buf, self._give, blk)
        return np.frombuffer(buf, dtype=dtype).reshape(shape, order=order)

    def _give(self, blk):
        try:
            if self.enabled and sum(b[0] for b in self.free) + blk[0] <= self.MAX_IDLE:
                self.free.append(blk)
            else:
                load().proxtv_host_free(C.c_void_p(blk[1]))
        except Exception:        # interpreter shutdown
            pass

    def clear(self):
        lib = load()
        for b in self.free:
            lib.proxtv_host_free(C.c_void_p(b[1]))
        self.free = []


_pool = _PinnedPool()


def set_pinned_results(on):
    """Results of at least 1 MiB come from a pool of page-locked host blocks (default: on); returns the previous setting."""
    prev = _pool.enabled
    _pool.enabled = bool(on)
    if not on:
        _pool.clear()
    return prev


# ======================================================================================================================
# 1D
# ======================================================================================================================
_TV1_METHODS = ("classictautstring", "linearizedtautstring", "hybridtautstring", "pn", "condat", "dp",
                "condattautstring", "kolmogorov")      # prox_tv/__init__.py:163-172


def tv1_1d(x, w, method="hybridtautstring", sigma=0.05, maxbacktracks=None):
    r"""1D TV-L1 prox: argmin_y 0.5||x-y||^2 + w sum_i |y_i - y_{i+1}|   (prox_tv/__init__.py:124-178).

    Every ``method`` of the reference computes the same unique minimiser; here they all run the exact linearized
    taut-string scan on the GPU (bit-identical to the reference's 'linearizedtautstring' and, whenever its backtracking
    budget is not exhausted, to its default 'hybridtautstring').  ``sigma`` / ``maxbacktracks`` are accepted and ignored.
    Returns a flat float64 array of ``np.size(x)`` elements, like the reference.
    """
    assert method in _TV1_METHODS
    assert w >= 0
    w = force_float_scalar(w)
    x = force_float_matrix(x)
    y = np.zeros(np.size(x))
    if x.size:
        xin = x if x.flags.c_contiguous or x.flags.f_contiguous else np.ascontiguousarray(x)
        _host_call("prox_fibers", y, xin, y, 1, int(np.size(x)), 1, w, None)
    return y


def tv1w_1d(x, w, method="tautstring", sigma=0.05):
    r"""Weighted 1D TV-L1 prox: argmin_y 0.5||x-y||^2 + sum_i w_i |y_i - y_{i+1}|   (prox_tv/__init__.py:218-254).

    Both reference methods ('tautstring', 'pn') compute the same minimiser; the GPU path is the weighted taut-string
    scan, bit-identical to the reference's 'tautstring'.
    """
    assert np.all(w >= 0)
    assert np.size(x) - 1 == np.size(w)
    w = force_float_matrix(w)
    x = force_float_matrix(x)
    y = np.zeros(np.size(x))
    n = int(np.size(x))
    if n == 1:
        y[0] = x.ravel()[0]
    elif n > 1:
        _host_call("prox_fibers", y, np.ascontiguousarray(x), y, 1, n, 1, 0.0, np.ascontiguousarray(w))
    return y


def _prox_rows(x, w, wt):
    """The device prox of every row of the contiguous float32/float64 CUDA tensor x (B, L); penalty w, or weights wt (B, L-1)."""
    import torch
    out = torch.empty_like(x)
    _dev_call("prox_fibers_dev", x, x, out, x.shape[0], x.shape[1], 1, w, wt)
    return out


def _batched_1d(x, w, weights):
    """x: (B, L) numpy array or torch CUDA tensor, row-contiguous signals.  w: float, or (torch path) a 0-dim tensor."""
    if _is_torch(x):
        import torch
        assert x.is_cuda and x.dim() == 2
        xt = x.contiguous()
        f32 = xt.dtype == torch.float32
        if not f32 and xt.dtype != torch.float64:
            xt = xt.double()
        B, L = xt.shape
        wt = None
        if weights is not None:
            wt = weights.to(dtype=xt.dtype, device=xt.device).contiguous()
            assert tuple(wt.shape) == (B, L - 1)
        wf, w_t = _w_float(w)
        if _needs_grad(xt, wt, w_t):
            return _autograd().ProxRows.apply(xt, wf, w_t, wt)
        return _prox_rows(xt, wf, wt)
    x = np.asarray(x)
    assert x.ndim == 2
    f32 = x.dtype == np.float32
    x = np.ascontiguousarray(x, dtype=np.float32 if f32 else np.float64)
    B, L = x.shape
    out = np.empty_like(x)
    wv = None
    if weights is not None:
        wv = np.ascontiguousarray(weights, dtype=x.dtype)
        assert wv.shape == (B, L - 1)
        assert np.all(wv >= 0)
    if x.size:
        _host_call("prox_fibers", x, x, out, B, L, 1, float(w), wv)
    return out


def tv1_1d_batched(x, w):
    """``tv1_1d`` on every row of a (B, L) array (numpy float64/float32, or a torch CUDA tensor).

    torch: differentiable.  With grad mode on and ``x`` or ``w`` requiring grad, the result carries a ``grad_fn`` whose backward is the
    exact vector-Jacobian product of the prox (proxtv_prox_fibers_vjp_dev_*: every sample gets the mean of the upstream gradient over
    its constant segment), run on the current CUDA stream; double backward is not supported.  ``w`` may be a float or a 0-dim tensor;
    a tensor's gradient is the sum of the per-edge gradients, accumulated in float64.  The forward result is the same either way.
    """
    assert w >= 0
    return _batched_1d(x, w if _is_torch(w) else float(w), None)


def tv1w_1d_batched(x, w):
    """``tv1w_1d`` on every row of x (B, L) with per-edge weights w (B, L-1)  -- BASELINE config 3.

    torch: differentiable with respect to ``x`` and the weights tensor ``w`` (see ``tv1_1d_batched``); a zero weight never fuses its
    edge, so its gradient is the signed difference of the two sides' gradients like any other edge between segments.
    """
    return _batched_1d(x, 0.0, w)


# ======================================================================================================================
# 2D
# ======================================================================================================================
_TV1_2D_METHODS = ("yang", "dr", "pd", "kolmogorov", "condat", "chambolle-pock", "chambolle-pock-acc")  # :391-399
_CP2_ALGS = {"condat": 0, "chambolle-pock": 1, "chambolle-pock-acc": 2}                          # the `alg` of CondatChambollePock2_TV
_CP2W_ALGS = {"condat": 0, "chambolle-pock": 1}          # the weighted solver's `alg` (proxtv_CP2W_TV_*)
_TV1_2D_GPU_METHODS = ("dr", "pd") + tuple(_CP2_ALGS)


def tv1_2d(x, w, n_threads=1, max_iters=0, method="dr", backward=None):
    r"""2D anisotropic TV-L1 prox (prox_tv/__init__.py:355-416).

    ``method='dr'`` (default) reproduces the reference's DR2_TV iteration exactly (35 fixed iterations unless
    ``max_iters`` > 0 -- NOT a converged solve, see SURVEY.md section 0.3); ``'pd'`` reproduces PD2_TV.  ``'condat'``,
    ``'chambolle-pock'`` and ``'chambolle-pock-acc'`` reproduce CondatChambollePock2_TV bit for bit (float64): primal-dual
    iterations run until X stops changing or ``max_iters`` (0: 2500) -- the converged prox (DESIGN.md section 15); by default they
    have no backward pass (see ``backward``).  ``'yang'`` and ``'kolmogorov'`` are not provided.  ``n_threads`` is ignored.
    numpy input: returns a Fortran-ordered float64 array like the reference.  torch CUDA tensor input (2D, float64 or
    float32): stays on the device and returns a tensor of the same dtype/layout.

    torch: differentiable with respect to ``x`` and ``w`` given as a 0-dim tensor.  With grad mode on and one of them requiring
    grad, the forward records a segmentation tape of every prox pass (2 bits per element per pass, kept on the device until the
    backward) and the backward is the exact vector-Jacobian product of the fixed 35-iteration splitting that is computed
    (proxtv_DR2_TV_vjp_dev_*, DESIGN.md section 11), run on the current CUDA stream; double backward is not supported.
    ``method='pd'`` on a tensor is ``tvgen(x, [w, w], [1, 2], [1, 1], max_iters=max_iters)`` on it (PD2_TV, same code, same
    gradients; the gradient of ``w`` is the sum of both terms' penalty gradients, in float64).

    ``backward='converged'`` (``'condat'`` and ``'chambolle-pock'`` only, opt-in): torch tensors become differentiable with respect to
    ``x`` and ``w`` given as a 0-dim tensor through the Jacobian of the prox itself, not of the iterations computed: the result is
    constant on clusters of pixels joined by fused edges (DESIGN.md section 15.2), the gradient of ``x`` is the upstream gradient
    averaged over each cluster and that of ``w`` sums sgn(y_j - y_i) (gx_i - gx_j) over the cut edges.  The forward records a fused-edge
    tape (2 bits per element) after its last iteration and returns the same bits as an unrecorded solve.  This gradient is right only
    when the forward has converged (it stopped before ``max_iters``, or at least reached the prox's partition of fused edges); the
    accelerated ``'chambolle-pock-acc'`` does not reach it and is refused, as are ``'dr'`` and ``'pd'``, which have their own exact
    backward.  Double backward is not supported; numpy input is unaffected.
    """
    assert w >= 0
    assert method in _TV1_2D_METHODS
    if method not in _TV1_2D_GPU_METHODS:
        raise NotImplementedError("proxtv_b200 implements the 2D solvers %s; got %r" % (", ".join(map(repr, _TV1_2D_GPU_METHODS)), method))
    _converged_backward(method, backward)
    if method == "pd":
        if _is_torch(x):
            assert x.dim() == 2
            assert not _is_torch(w) or w.dim() == 0, "w must be a number or a 0-dim tensor"
            wf, w_t = _w_float(w)
            return _nd_torch("PD2_TV", tvgen, x, [wf, wf], w_t, [1, 2], max_iters)
        x = np.asfortranarray(x, dtype="float64")
        assert x.ndim == 2
        w = force_float_scalar(w)
        y = _pool.empty(x.shape, np.float64, "F")
        info = np.zeros(_N_INFO)
        _host_call("PD2_TV", None, x, np.array([w, w]), np.array([1.0, 1.0]), np.array([1.0, 2.0]), y, info,
                   np.array(x.shape, dtype=np.int32), 2, 2, int(n_threads), int(max_iters), info=info)
        return y
    return _tv2(x, w, max_iters, method, batched=False, backward=backward)


def tv1w_2d(x, w_col, w_row, max_iters=0, n_threads=1, method="dr", backward=None):
    r"""2D weighted anisotropic TV-L1 prox by Douglas-Rachford splitting (prox_tv/__init__.py:445-481 -> DR2L1W_TV).

    ``w_col``: (M-1, N) weights of the differences along columns, ``w_row``: (M, N-1) along rows.  Same fixed-iteration
    scheme as ``tv1_2d(method='dr')`` (35 iterations unless ``max_iters`` > 0).  ``n_threads`` is ignored.
    numpy input: Fortran-ordered float64 result like the reference.  torch CUDA tensors (float64 / float32, weights of any
    floating dtype on any device): computed on x's device, returns a tensor shaped and typed like ``x``.

    ``method='condat'`` or ``'chambolle-pock'``: the converged weighted prox instead, the primal-dual iteration of
    ``tv1_2d(method=...)`` with each dual clipped to its own edge's weight, run until X stops changing or ``max_iters`` (0: 2500)
    (proxtv_CP2W_TV_*, DESIGN.md section 15.1).  With every weight equal to w it is ``tv1_2d(x, w, method=...)`` bit for bit in
    float64.  torch tensors of either memory order are solved in place of their layout and the result has the solved tensor's
    layout; by default these methods have no backward pass.  ``'chambolle-pock-acc'`` is not available: its step rule needs one penalty.
    ``backward='converged'`` (opt-in, these two methods only) makes them differentiable on torch tensors with respect to ``x``,
    ``w_col`` and ``w_row`` through the Jacobian of the prox at the partition the forward reached, as ``tv1_2d(backward='converged')``
    describes: each edge weight gets sgn(y_j - y_i) (gx_i - gx_j) on a cut edge and 0 on a fused one.  Right only when the forward has
    converged; weights of another dtype or device, and expanded weights, get their gradients through ordinary autograd.

    torch: differentiable with respect to ``x``, ``w_col`` and ``w_row``.  With grad mode on and one of them requiring grad, the
    forward records a segmentation tape of every prox pass (2 bits per element per pass, kept on the device until the backward) and
    the backward is the exact vector-Jacobian product of the fixed-iteration splitting that is computed (proxtv_DR2L1W_TV_vjp_dev_*,
    DESIGN.md section 12), run on the current CUDA stream; each edge weight gets its own gradient.  Weights of another dtype or
    device, and expanded weights (``w.expand(M - 1, N)``), get theirs through ordinary autograd.  The forward result is the same
    either way; double backward is not supported.
    """
    _converged_backward(method, backward)
    _w2_method(method)
    if method != "dr":
        return _tv2w(x, w_col, w_row, max_iters, method, batched=False, backward=backward)
    if _is_torch(x):
        return _drw_torch(x, w_col, w_row, max_iters)
    assert np.all(np.asarray(w_col) >= 0)             # the reference's checks in its order: an x that is not 2D raises ValueError
    assert np.all(np.asarray(w_row) >= 0)
    M, N = np.shape(x)
    assert np.shape(w_col) == (M - 1, N)
    assert np.shape(w_row) == (M, N - 1)
    return _tv2w_numpy(x, w_col, w_row, max_iters, None, batched=False)


def _drw_torch(x, w_col, w_row, max_iters):
    """The torch path of tv1w_2d(method='dr'); recorded by the Function when grad mode is on and x, w_col or w_row requires grad.  The
    solver works on column-major arrays, the row-major storage of the transposes: the transposes and casts to them are ordinary autograd
    ops."""
    import torch
    assert x.is_cuda and x.dtype in (torch.float64, torch.float32) and x.dim() == 2
    M, N = int(x.shape[0]), int(x.shape[1])
    assert tuple(w_col.shape) == (M - 1, N) and tuple(w_row.shape) == (M, N - 1)
    xt = x.t().contiguous()
    w1 = w_col.to(device=x.device, dtype=x.dtype).t().contiguous()
    w2 = w_row.to(device=x.device, dtype=x.dtype).t().contiguous()
    geom = (M, N, 1, 0, None, int(max_iters))
    if _needs_grad(x, w_col, w_row):
        return _autograd().TV2.apply(xt, w1, w2, 0.0, None, "DR2L1W_TV_batched", geom).t()
    return _tv2_solve("DR2L1W_TV_batched", xt, w1, w2, 0.0, geom).t()


def tv1w_2d_batched(x, w_col, w_row, max_iters=0, method="dr", backward=None):
    r"""``tv1w_2d`` on every image of x (B, H, W), with per-image weight maps ``w_col`` (B, H-1, W) (edges along columns) and
    ``w_row`` (B, H, W-1) (edges along rows).  Each image is solved independently with exactly the single-image iteration (its own
    2 * mean start value, 35 iterations unless ``max_iters`` > 0).

    numpy: float64, or float32 solved in float32; the weights are cast to x's dtype.  Returns a C-ordered (B, H, W) array of x's dtype.
    torch: a CUDA tensor (float32 / float64).  C-ordered and per-image column-major tensors are solved in place of their layout (no
    transposes), anything else is made contiguous; the result has the solved tensor's layout.  Weights of any floating dtype or
    device are moved to x's device and dtype and laid out like it through ordinary autograd ops.  Differentiable with respect to
    ``x``, ``w_col`` and ``w_row`` like ``tv1w_2d`` (proxtv_DR2L1W_TV_batched_vjp_dev_*, DESIGN.md section 12); an expanded weight
    (``w.expand(B, H - 1, W)``) gets the sum of its per-edge gradients through autograd.

    ``method='condat'`` or ``'chambolle-pock'``: the converged weighted prox of ``tv1w_2d(method=...)`` on every image, each running
    until its own stop test holds (float32: float32 arithmetic).  Results as above (numpy: C-ordered, x's dtype; torch: the solved
    tensor's layout); no backward pass unless ``backward='converged'``, the opt-in gradient of ``tv1w_2d``, per image.
    """
    _converged_backward(method, backward)
    _w2_method(method)
    return _tv2w(x, w_col, w_row, max_iters, method, batched=True, backward=backward)


def _drw_lay(w, xin, row_major):
    """A weight map (or a batch of them) on xin's device and dtype, laid out like xin's images (row_major = 1: C order; 0: every map
    column-major), through ordinary autograd ops."""
    w = w.to(device=xin.device, dtype=xin.dtype)
    return w.contiguous() if row_major else w.transpose(-2, -1).contiguous().transpose(-2, -1)


def _dr2_layout(x, batched):
    """(M, N, batch, row_major, xin) of a 2D / batched 3D CUDA tensor: either memory order of the trailing two dims is taken as it
    is, anything else is copied to C order."""
    import torch
    assert x.is_cuda and x.dtype in (torch.float64, torch.float32)
    assert x.dim() == (3 if batched else 2)
    M, N = int(x.shape[-2]), int(x.shape[-1])
    batch = int(x.shape[0]) if batched else 1
    # accept either memory order of the trailing two dims without copying
    if x.stride(-1) == 1 and x.stride(-2) == N and (not batched or x.stride(0) == M * N):
        row_major, xin = 1, x
    elif x.stride(-2) == 1 and x.stride(-1) == M and (not batched or x.stride(0) == M * N):
        row_major, xin = 0, x
    else:
        row_major, xin = 1, x.contiguous()
    return M, N, batch, row_major, xin


def tv1_2d_batched(x, w, max_iters=0, method="dr", backward=None):
    """``tv1_2d(method=method)`` on every image of x (B, H, W)  -- BASELINE config 5 with the default ``method='dr'``.

    numpy: float64 or float32, C-ordered (B, H, W); torch: CUDA tensor (B, H, W).  Each image is solved independently with
    exactly the single-image iteration (its own 2*mean initialisation).  torch: differentiable like ``tv1_2d``.
    ``method`` 'condat', 'chambolle-pock' or 'chambolle-pock-acc': each image runs until its own stop test holds (float32: float32
    arithmetic); numpy results are C-ordered arrays of x's dtype, tensors keep their layout; no backward pass unless
    ``backward='converged'`` ('condat' and 'chambolle-pock'), the opt-in gradient of ``tv1_2d``, per image (the gradient of a 0-dim
    ``w`` sums every image's).
    """
    assert w >= 0
    assert method == "dr" or method in _CP2_ALGS, "method must be 'dr', 'condat', 'chambolle-pock' or 'chambolle-pock-acc'"
    _converged_backward(method, backward)
    return _tv2(x, w, max_iters, method, batched=True, backward=backward)


def _converged_backward(method, backward):
    """Validates the ``backward`` keyword of the 2D solvers: None, or 'converged' with 'condat' / 'chambolle-pock'."""
    assert backward in (None, "converged"), "backward must be None or 'converged'"
    if backward == "converged" and method not in _CP2W_ALGS:
        why = ("does not reach the prox's partition of fused edges in its iterations" if method == "chambolle-pock-acc"
               else "is a fixed splitting with its own exact backward (omit backward=)")
        raise NotImplementedError("backward='converged' is the Jacobian of the converged prox, for method 'condat' or 'chambolle-pock'; "
                                  "method %r %s" % (method, why))


def _w2_method(method):
    """Validates the method of the weighted 2D prox: 'dr', 'condat' or 'chambolle-pock'."""
    if method == "chambolle-pock-acc":
        raise NotImplementedError("the weighted 2D prox has no 'chambolle-pock-acc': its accelerated step rule takes gamma = 1 / lambda "
                                  "from one penalty, and per-edge weights give none; use 'condat' or 'chambolle-pock'")
    assert method == "dr" or method in _CP2W_ALGS, "method must be 'dr', 'condat' or 'chambolle-pock'"


def _tv2(x, w, max_iters, method, batched, backward=None):
    """tv1_2d / tv1_2d_batched with method 'dr' (DR2_TV) or a primal-dual one (CP2_TV, alg _CP2_ALGS[method]).  numpy: _tv2_numpy;
    torch: either memory order (_dr2_layout), result in the solved tensor's layout."""
    alg = _CP2_ALGS.get(method)
    if not _is_torch(x):
        return _tv2_numpy(x, w, max_iters, alg, batched)
    if alg is not None and _needs_grad(x, w) and backward is None:
        raise NotImplementedError("tv1_2d method %r has no backward pass by default; pass backward='converged' for the Jacobian of "
                                  "the converged prox, use method='dr' or 'pd' for gradients, or call it under torch.no_grad() / "
                                  "on a detached tensor" % method)
    entry = "DR2_TV" if alg is None else "CP2_TV"
    wf, w_t = _w_float(w)
    M, N, batch, row_major, xin = _dr2_layout(x, batched)
    geom = (M, N, batch, row_major, alg, int(max_iters))
    if _needs_grad(x, w_t):
        return _autograd().TV2.apply(xin, None, None, wf, w_t, entry, geom)
    return _tv2_solve(entry, xin, None, None, wf, geom)


def _tv2w(x, w_col, w_row, max_iters, method, batched, backward=None):
    """tv1w_2d_batched, and tv1w_2d's primal-dual methods: 'dr' (DR2L1W_TV) or a primal-dual method (CP2W_TV, alg _CP2W_ALGS[method]).
    numpy: _tv2w_numpy; torch: either memory order (_dr2_layout), the weight maps laid out to match, result in the solved tensor's
    layout."""
    alg = _CP2W_ALGS.get(method)
    cp = alg is not None
    if not _is_torch(x):
        x = np.asarray(x)
        assert x.ndim == (3 if batched else 2)
        assert np.all(np.asarray(w_col) >= 0)
        assert np.all(np.asarray(w_row) >= 0)
        lead, (M, N) = x.shape[:-2], x.shape[-2:]
        assert np.shape(w_col) == lead + (M - 1, N)
        assert np.shape(w_row) == lead + (M, N - 1)
        return _tv2w_numpy(x, w_col, w_row, max_iters, alg, batched)
    if cp and _needs_grad(x, w_col, w_row) and backward is None:
        raise NotImplementedError("tv1w_2d method %r has no backward pass by default; pass backward='converged' for the Jacobian of "
                                  "the converged prox, use method='dr' for gradients, or call it under torch.no_grad() / on "
                                  "detached tensors" % method)
    entry = "CP2W_TV" if cp else "DR2L1W_TV_batched"
    M, N, batch, row_major, xin = _dr2_layout(x, batched)
    lead = (batch,) if batched else ()
    assert tuple(w_col.shape) == lead + (M - 1, N) and tuple(w_row.shape) == lead + (M, N - 1)
    w1, w2 = _drw_lay(w_col, xin, row_major), _drw_lay(w_row, xin, row_major)
    geom = (M, N, batch, row_major, alg, int(max_iters))
    if _needs_grad(x, w_col, w_row):
        return _autograd().TV2.apply(xin, w1, w2, 0.0, None, entry, geom)
    return _tv2_solve(entry, xin, w1, w2, 0.0, geom)


def _host_images(x, batched, transposed=False):
    """(x, out, M, N, batch, row_major): a numpy image or batch of images laid out as the host 2D entry points take it, and a result
    array from the pool in the same layout.  One image: a Fortran-ordered float64 copy, a column-major batch of one (row_major = 0).  A
    batch (B, M, N): float32 kept, anything else float64, C-ordered (row_major = 1) -- or, transposed, the C-ordered (B, N, M) array of
    its transposes, which is the column-major images back to back (row_major = 0)."""
    if not batched:
        x = np.asfortranarray(x, dtype="float64")
        assert x.ndim == 2
        return (x, _pool.empty(x.shape, np.float64, "F")) + x.shape + (1, 0)
    x = np.asarray(x)
    assert x.ndim == 3
    dt = np.float32 if x.dtype == np.float32 else np.float64
    B, M, N = x.shape
    x = np.ascontiguousarray(np.transpose(x, (0, 2, 1)) if transposed else x, dtype=dt)
    return x, _pool.empty(x.shape, dt, "C"), M, N, B, 0 if transposed else 1


def _tv2_numpy(x, w, max_iters, alg, batched):
    """The numpy solve of tv1_2d / tv1_2d_batched: 'dr' (alg None) through proxtv_DR2_TV_batched_*, which returns 0 on success and takes
    column-major images only (a batch is solved as its transposes and the result transposed back); the primal-dual methods through
    proxtv_CP2_TV_batched_*, which an empty batch does not reach.  One image: Fortran-ordered float64 result; a batch: x's dtype."""
    w = force_float_scalar(w)
    x, out, M, N, B, row_major = _host_images(x, batched, transposed=alg is None)
    info = np.zeros(_N_INFO * max(B, 1))
    if alg is None:
        _host_call("DR2_TV_batched", x, M, N, B, x, w, w, out, int(max_iters), info, rc=False, info=info)
        return np.transpose(out, (0, 2, 1)) if batched else out
    if x.size or not batched:
        _host_call("CP2_TV_batched", x, M, N, B, row_major, x, w, out, alg, int(max_iters), info, info=info)
    return out


def _tv2w_numpy(x, w_col, w_row, max_iters, alg, batched):
    """The numpy solve of tv1w_2d / tv1w_2d_batched on checked input: 'dr' (alg None) through proxtv_DR2L1W_TV_batched_*, which returns 0
    on success, the primal-dual methods through proxtv_CP2W_TV_batched_*; the weight maps laid out like the images (_host_images), and
    an empty batch reaches neither.  One image: Fortran-ordered float64 result; a batch: C-ordered, x's dtype."""
    x, out, M, N, B, row_major = _host_images(x, batched)
    order = "C" if row_major else "F"
    w1, w2 = (np.require(np.asarray(w), x.dtype, [order]) for w in (w_col, w_row))
    if x.size:
        info = np.zeros(_N_INFO * B)
        entry, alg_ = ("DR2L1W_TV_batched", ()) if alg is None else ("CP2W_TV_batched", (alg,))
        _host_call(entry, x, M, N, B, row_major, x, w1, w2, out, *alg_, int(max_iters), info, rc=alg is not None, info=info)
    return out


# The taped 2D solvers, by entry point (proxtv_<entry>_dev_* / _record_dev_* / _vjp_dev_*): the tape size, and whether the entry is a
# Douglas-Rachford one.  Those take the tape before info when recording and (maxit, tape) in the backward, and their unrecorded solve
# returns 0 on success like the reference's; the primal-dual ones take an alg, the tape after info and (tape, X) in the backward -- so
# their result is saved for it -- and return 1.
_TAPED = {
    "DR2_TV": (lambda lib, M, N, batch, maxit: lib.proxtv_DR2_TV_tape_bytes(M, N, batch, maxit), True),
    "DR2L1W_TV_batched": (lambda lib, M, N, batch, maxit: lib.proxtv_DR2L1W_TV_batched_tape_bytes(M, N, batch, maxit), True),
    "CP2_TV": (lambda lib, M, N, batch, maxit: lib.proxtv_CP2_TV_tape_bytes(M, N, batch), False),
    "CP2W_TV": (lambda lib, M, N, batch, maxit: lib.proxtv_CP2_TV_tape_bytes(M, N, batch), False),
}


def _tv2_solve(entry, xin, W1, W2, w, geom, tape=None):
    """proxtv_<entry>_dev_* (a _TAPED entry) on xin, geom = (M, N, batch, row_major, alg, max_iters), alg None for the Douglas-Rachford
    entries: with the weight maps W1, W2 laid out like xin, else the penalty w; given a tape (a uint8 CUDA tensor of the entry's tape
    size) the _record_dev_ form, the same solve recording its tape.  The result has xin's layout."""
    import torch
    M, N, batch, row_major, alg, max_iters = geom
    dr = _TAPED[entry][1]
    out = torch.empty_strided(xin.shape, xin.stride(), dtype=xin.dtype, device=xin.device)
    info = np.zeros(_N_INFO * max(batch, 1))
    pen = (W1, W2) if W1 is not None else (w, w) if dr else (w,)
    args = (M, N, batch, row_major, xin, *pen, out) + (() if dr else (alg,)) + (max_iters,)
    if tape is None:
        _dev_call(entry + "_dev", xin, *args, info, rc=not dr, info=info)
    else:
        rec = (tape, tape.numel(), info) if dr else (info, tape, tape.numel())
        _dev_call(entry + "_record_dev", xin, *args, *rec, info=info)
    return out


# ======================================================================================================================
# ND
# ======================================================================================================================
def tvgen(x, ws, ds, ps, n_threads=1, max_iters=0):
    r"""General ND TV prox with one 1D TV-L1 term per entry of (ws, ds, ps)   (prox_tv/__init__.py:533-600).

    Dispatch follows the reference, including its quirks: the DR2_TV branch of the reference is dead code
    (``len(ds) == 2 & ds[0] == 1 & ds[1] == 2`` is always False, :585), so two terms go to PD2_TV and anything else to
    PD_TV.  PD_TV scales the caller's ``ws`` by ``len(ws)`` IN PLACE when ``ws`` is a float64 ndarray (:576 does not
    copy in that case; src/TVNDopt.cpp:100-101).  Only p = 1 norms are implemented on the GPU path.
    Extension: a float32 ``x`` is solved in float32 (the reference would upcast) when ``len(ws) != 2``.
    ``tvgen.last_info`` = [iterations, mean|x - x_last|, RC].  Both solvers stop when mean|x - x_last| <= 1e-6 or after
    ``max_iters`` iterations (0: 35).

    torch: ``x`` a CUDA tensor (float32 or float64, any ndim >= 1) is solved on its device and current stream with the same
    dispatch (two terms: PD2_TV, whatever ``ds`` is; else PD_TV), and the result is a tensor of x's shape and dtype, in x's memory
    order when x is C- or Fortran-contiguous (no copy is made: a C-ordered tensor is the column-major array of the reversed shape),
    else C order.  ``ds`` are 1-based axes of ``x``; an axis without a term is a batch axis, but the stop test is global, so the
    slices are solved independently only when the ``max_iters`` cap ends the solve (otherwise all stop together).  ``ws`` may be a
    list, an ndarray or a 1-D tensor of any float dtype and device, and is never modified on this path.
    Differentiable with respect to ``x`` and a ``ws`` tensor: with grad mode on and one of them requiring grad, the forward
    records the segmentation tape of every prox pass (2 bits per element per pass, kept on the device until the backward) and the
    backward is the exact vector-Jacobian product of the K iterations the forward ran (proxtv_PD_TV_vjp_dev_* /
    proxtv_PD2_TV_vjp_dev_*, DESIGN.md section 14), run on the current CUDA stream.  K is picked by the stop test and has no
    derivative of its own: where a perturbation changes K the computed map jumps.  The tape is allocated for ``max_iters``
    iterations, not for the ones that turn out to run, so a large ``max_iters`` costs its memory up front: PD_TV on a
    512 x 512 x 256 volume with 3 terms at 35 iterations is 105 passes x 16 MiB, about 1.64 GiB.  Double backward is not
    supported.  The forward result is the same either way.
    """
    return _tvgen_front(tvgen, False, x, ws, ds, ps, n_threads, max_iters)


tvgen.last_info = None


def _nd_checks(ws, ds, ps, max_iters, n_threads=1):
    assert len(ws) == len(ds)
    assert len(ws) == len(ps)
    assert n_threads >= 1
    assert max_iters >= 0


def _p1(ps):
    if np.any(force_float_matrix(ps) != 1):
        raise NotImplementedError("proxtv_b200 implements TV-L1 (p = 1) penalty terms only")


def _nd_solver(npen, pdr=False):
    """The solver of tvgen (two terms: PD2_TV, any other count: PD_TV) or, pdr, tvgen_pdr's PDR_TV."""
    return "PDR_TV" if pdr else "PD2_TV" if npen == 2 else "PD_TV"


def _tvgen_front(owner, pdr, x, ws, ds, ps, n_threads, max_iters):
    """tvgen (owner tvgen: the proximal Dykstra solvers) and tvgen_pdr (owner tvgen_pdr, pdr: PDR_TV).  numpy: the reference's symbol on
    a Fortran-ordered float64 copy -- float32 only where PD_TV has its own route, proxtv_PD_TV_f32 -- given ws itself when it is a
    float64 ndarray (PD_TV and PDR_TV scale it in place); sets owner.last_info.  torch: _nd_torch."""
    _nd_checks(ws, ds, ps, max_iters, n_threads)
    if _is_torch(x):
        _p1(ps)
        lam, ws_t = _ws_floats(ws)
        return _nd_torch(_nd_solver(len(lam), pdr), owner, x, lam, ws_t, ds, max_iters)
    solver = _nd_solver(len(ws), pdr)
    f32 = solver == "PD_TV" and isinstance(x, np.ndarray) and x.dtype == np.float32
    x = np.asfortranarray(x, dtype="float32" if f32 else "float64")
    ws = force_float_matrix(ws)
    ps = force_float_matrix(ps)
    _p1(ps)
    y = _pool.empty(np.shape(x), x.dtype, "F")
    info = np.zeros(_N_INFO)
    dsa = np.array(ds, dtype=np.float64)
    ns = np.array(x.shape, dtype=np.int32)
    if f32:
        _host_call("PD_TV", x, x, ws, dsa, y, info, ns, x.ndim, len(ws), int(max_iters), info=info)
    else:
        _host_call(solver, None, x, ws, ps, dsa, y, info, ns, x.ndim, len(ws), int(n_threads), int(max_iters), info=info)
    owner.last_info = info
    return y


def _f_contiguous(x):
    """True when the tensor's memory is the column-major (Fortran) order of its shape (axes of size 1 may have any stride)."""
    step = 1
    for n, st in zip(x.shape, x.stride()):
        if n != 1 and st != step:
            return False
        step *= n
    return True


def _nd_layout(x, ds, batched=False):
    """(ns, dims, xin) of an N-D CUDA tensor for the column-major solvers; batched: a batch of items along its first axis, ns and dims
    those of an item.  Items that are column-major and back to back (the batch axis slowest) are taken as they are, with their shape
    and axes; anything else is a C-ordered array (copied to C order unless it is one already), each item of which is the column-major
    array of its reversed shape (_pdr_c_order), so no transpose is made."""
    import torch
    assert x.is_cuda and x.dtype in (torch.float64, torch.float32) and x.dim() >= (2 if batched else 1)
    if not x.is_contiguous() and _f_contiguous(x.movedim(0, -1) if batched else x):
        return [int(n) for n in x.shape[batched:]], [float(d) for d in ds], x
    xin = x.contiguous()
    return _pdr_c_order(xin.shape[batched:], ds) + (xin,)


def _pdr_c_order(shape, ds):
    """(ns, dims) of the solver for a C-ordered array of this shape and 1-based axes ds: the reversed shape, axis a -> nds + 1 - a."""
    nd = len(shape)
    return [int(n) for n in shape][::-1], [float(nd + 1 - d) for d in ds]


def _ws_floats(ws):
    """(the penalties as a list of floats, ws when it is a tensor else None) of a list, ndarray or 1-D tensor; ws is not written."""
    if _is_torch(ws):
        import torch
        assert ws.dim() == 1, "ws must be a 1-D tensor of one penalty per term"
        return [float(v) for v in ws.detach().to(device="cpu", dtype=torch.float64).numpy()], ws
    return [float(v) for v in np.asarray(ws, dtype=np.float64).ravel()], None


def _ws_rows(ws):
    """ws as a float64 (rows, terms) ndarray when it has two dimensions (a nested list, an ndarray or a tensor: one row of penalties
    per item), else None; ws is not written."""
    if _is_torch(ws):
        import torch
        return ws.detach().to(device="cpu", dtype=torch.float64).numpy() if ws.dim() == 2 else None
    a = np.asarray(ws, dtype=np.float64)
    return a if a.ndim == 2 else None


def _nd_torch(solver, owner, x, lam, ws_t, ds, max_iters, batched=False, items=False):
    """The torch path of tvgen_pdr, tvgen, tv1_2d(method='pd') and (batched) tvgen_batched; recorded by the Function when grad mode is
    on and x, or the penalty tensor ws_t, requires grad.  lam: the penalties as floats; ws_t: None, a 1-D tensor of them, or a 0-dim
    tensor shared by every term.  items (batched): lam holds one row of len(ds) penalties per item, item-major, and ws_t is None or
    the (B, len(ds)) tensor of them.  Nothing the caller passed is written: the solve gets a float64 copy of lam, which PDR_TV and PD_TV
    scale in place.  Sets owner.last_info."""
    import torch
    rows = int(x.shape[0]) if items else 1
    assert len(lam) == rows * len(ds)
    assert ws_t is None or tuple(ws_t.shape) in (((rows, len(ds)),) if items else ((), (len(lam),))), \
        "ws must be one penalty per term, or one 0-dim penalty for all"
    ns, dims, xin = _nd_layout(x, ds, batched)
    batch = int(x.shape[0]) if batched else 0
    if batched and batch == 0:
        owner.last_info = np.zeros((0, _N_INFO))
        return torch.empty_like(x)
    args = (solver, np.array(ns, dtype=np.int32), np.array(dims, dtype=np.float64), np.array(lam, dtype=np.float64), int(max_iters),
            owner, batch, items)
    if _needs_grad(x, ws_t):
        return _autograd().ND.apply(xin, ws_t, *args)
    return _nd_solve(xin, *args)[0]


def _nd_solve(xin, solver, nsa, dsa, lama, max_iters, owner, batch=0, items=False, tape=None):
    """proxtv_<solver>_dev_* (solver: "PDR_TV", "PD_TV" or "PD2_TV") on xin, column-major over nsa (see _nd_layout), or given a tape
    (a uint8 CUDA tensor, proxtv_<solver>_tape_bytes() long) proxtv_<solver>_record_dev_*, the same solve recording every prox pass's
    segmentation.  batch >= 1 (PD_TV / PD2_TV): xin holds `batch` items over nsa back to back, solved by proxtv_<solver>_batched_dev_* /
    _batched_record_dev_* (items: lama holds one row per item, proxtv_<solver>_batched_items_*), and info is (batch, 3).  Sets
    owner.last_info; returns (result in xin's layout, info)."""
    import torch
    out = torch.empty_strided(xin.shape, xin.stride(), dtype=xin.dtype, device=xin.device)
    info = np.zeros(_N_INFO * max(batch, 1))
    bat = (batch,) if batch else ()
    kind = ("_batched_items" if items else "_batched") if batch else ""
    args = (xin, lama, dsa, out, info, nsa, len(nsa), len(dsa)) + bat + (max_iters,)
    if tape is None:
        _dev_call(solver + kind + "_dev", xin, *args, info=info)
    else:
        _dev_call(solver + kind + "_record_dev", xin, *args, tape, tape.numel(), info=info)
    if batch:
        info = info.reshape(batch, _N_INFO)
    owner.last_info = info
    return out, info


def tvgen_batched(x, ws, ds, ps, max_iters=0):
    r"""``tvgen`` over a batch: x of shape (B, \*s) holds B independent items of shape s, and item b is solved as ``tvgen(x[b], ws, ds,
    ps, max_iters=max_iters)`` would solve it, with its own stop test.

    ``ds`` are 1-based axes of an item (1..len(s)); two terms go to PD2_TV and any other count to PD_TV, as in ``tvgen``; p = 1 terms
    only (anything else raises NotImplementedError).  ``ws`` is never written (``tvgen``'s in-place scaling of a float64 ndarray is not
    carried over) and is either shared by every item -- a list, an ndarray, a 1-D tensor or a 0-dim tensor, whatever B is -- or holds
    one row of penalties per item: a nested list, a 2-D ndarray or a 2-D tensor of shape (B, len(ds)), row b item b's penalties in
    ``ds`` order, so that item b is solved as ``tvgen(x[b], ws[b], ds, ps, max_iters=max_iters)`` would solve it
    (``proxtv_PD*_TV_batched_items_*``, DESIGN.md section 16.1).  Any other shape raises AssertionError before any device work.  Rows
    that are all equal give the shared call's result bit for bit.
    Per-item stop rule: item b iterates while mean|x_b - x_b,last| > 1e-6 and it < ``max_iters`` (0: 35) -- PD2_TV with one term runs
    one iteration -- so an item's result does not depend on the rest of the batch, and an item that has stopped costs no more prox
    work.  ``tvgen_batched.last_info`` is a (B, 3) array, row b = [K_b, stop_b, RC_b] as ``tvgen.last_info`` gives it for that item.
    Under the bit-faithful engines (``set_engine('seq')`` / ``'chunked'``) every item's result and info row equal the single-item
    solve of that item (``proxtv_PD*_TV_dev_*`` into an aligned buffer) bit for bit, in float64 and float32, whatever B is, wherever
    the item sits and whenever the others stop.  Under ``'auto'`` and ``'lane'`` the fiber route and the lane engine's suitability test
    are decided once for the whole batch (its fiber count, its first 2^18 elements), so an item's bits can differ from its single
    solve's (the lane engine computes in slope form); the results agree to about 1e-12 relative.
    numpy: float64, or float32 solved in float32, with both solvers; items are solved in column-major order, so item b is bit for bit
    ``tvgen(x[b], ...)`` under ``'chunked'``; returns a (B, \*s) array of x's dtype.
    torch: a CUDA tensor (float32 or float64, ndim >= 2) is solved on its device and current stream.  A C-ordered tensor is taken as
    it is (each item is the column-major array of its reversed shape), and so is one whose items are column-major and contiguous with
    the batch axis slowest; anything else is made C-contiguous; the result has the solved tensor's layout.  Differentiable with
    respect to x and a ``ws`` tensor: the forward records the segmentation tape of every prox pass and each item's K, and the backward
    is, for every item, the exact vector-Jacobian product of the K_b iterations that item ran (``proxtv_PD*_TV_batched_vjp_dev_*``,
    DESIGN.md section 16); the gradient of a shared ``ws`` tensor is the per-item penalty gradients summed in float64, that of a
    (B, len(ds)) one is row b = item b's penalty gradients (an expanded ``w.expand(B, npen)`` thus gives ``w`` their sum through
    autograd), each cast to the tensor's dtype and device.  K_b has no derivative: where a
    perturbation changes it the map jumps.  The tape is allocated for ``max_iters`` iterations of the whole batch, B times the single
    capacity: PD_TV with 3 terms at 35 iterations takes about 1.64 GiB per 512 x 512 x 256 item.  Double backward is not supported.
    """
    rows = _ws_rows(ws)
    if rows is None:
        _nd_checks(ws, ds, ps, max_iters)
        lam, ws_t = _ws_floats(ws)
        assert ws_t is None or tuple(ws_t.shape) in ((), (len(lam),)), "ws must be one penalty per term, or one 0-dim penalty for all"
    else:
        assert len(ds) == len(ps) and max_iters >= 0
        assert len(np.shape(x)) >= 2 and rows.shape == (int(np.shape(x)[0]), len(ds)), \
            "a 2-D ws must be (B, len(ds)): one row of penalties per item"
        lam, ws_t = [float(v) for v in rows.ravel()], (ws if _is_torch(ws) else None)
    _p1(ps)
    items = rows is not None
    solver = _nd_solver(len(ds))
    if _is_torch(x):
        return _nd_torch(solver, tvgen_batched, x, lam, ws_t, ds, max_iters, batched=True, items=items)
    x = np.asarray(x)
    f32 = x.dtype == np.float32
    assert x.ndim >= 2
    B = x.shape[0]
    if B == 0:
        tvgen_batched.last_info = np.zeros((0, _N_INFO))
        return np.zeros(x.shape, dtype=np.float32 if f32 else np.float64)
    rev = (0,) + tuple(range(x.ndim - 1, 0, -1))                    # (B, s_k .. s_1) in C order: every item column-major
    xt = np.ascontiguousarray(np.transpose(x, rev), dtype=np.float32 if f32 else np.float64)
    out = np.empty_like(xt)
    info = np.zeros(_N_INFO * B)
    ns = np.array(x.shape[1:], dtype=np.int32)
    lama = np.array(lam, dtype=np.float64)
    _host_call(solver + ("_batched_items" if items else "_batched"), xt, xt, lama, np.array(ds, dtype=np.float64), out, info, ns, len(ns),
               len(ds), B, int(max_iters), info=info)
    tvgen_batched.last_info = info.reshape(B, _N_INFO)
    return np.transpose(out, rev)


tvgen_batched.last_info = None


def tvgen_pdr(x, ws, ds, ps, n_threads=1, max_iters=0):
    r"""The same generalized TV prox as ``tvgen`` solved with the reference's Parallel Douglas-Rachford splitting, ``PDR_TV``
    (src/TVNDopt.cpp:280-500; reached from MATLAB only in the reference, matlab/solveTVND_PDR.cpp:89 -- SURVEY.md 8f N4).

    Runs exactly ``max_iters`` iterations (0: 35; the reference's loop has no stop test) and, like PD_TV, scales a float64
    ndarray ``ws`` by ``len(ws)`` IN PLACE.  float64 only from numpy; p = 1 norms only.
    ``tvgen_pdr.last_info`` = [iterations, mean|x - x_last|, RC].

    torch: ``x`` a CUDA tensor (float32 or float64, any ndim >= 1) is solved on its device and current stream and the result is a
    tensor of x's shape and dtype, in x's memory order when x is C- or Fortran-contiguous (no copy is made: a C-ordered tensor is the
    column-major array of the reversed shape), else C order.  ``ds`` are 1-based axes of ``x`` as on the numpy path; an axis without
    a term is a free batch axis.  ``ws`` may be a list, an ndarray or a 1-D tensor of any float dtype and device, and is never
    modified on this path.  Differentiable with respect to ``x`` and a ``ws`` tensor: with grad mode on and one of them requiring
    grad, the forward records the segmentation tape of every prox pass that reaches the result (2 bits per element per pass, kept
    on the device until the backward: 1.6 GiB for a 512 x 512 x 256 volume with 3 terms at 35 iterations) and the backward is the
    exact vector-Jacobian product of the fixed-iteration splitting that is computed (proxtv_PDR_TV_vjp_dev_*, DESIGN.md section 13),
    run on the current CUDA stream; double backward is not supported.  The forward result is the same either way.
    """
    return _tvgen_front(tvgen_pdr, True, x, ws, ds, ps, n_threads, max_iters)


tvgen_pdr.last_info = None


# ======================================================================================================================
# torch autograd
# ======================================================================================================================
@functools.cache
def _autograd():
    """The torch.autograd.Function of each differentiable solver, made on first use so that numpy users never import torch.

    Each forward is the solver's no-grad solve, given a tape by the iterative solvers; each backward runs the solver's vector-Jacobian
    product entry point on the current stream and returns None for an input that needs no gradient.  A penalty given as a float
    comes with the tensor it was read from (w_t / ws_t, or None), which only receives the gradient.  Double backward is not
    supported."""
    import torch
    from torch.autograd.function import once_differentiable

    class ProxRows(torch.autograd.Function):
        """apply(x, w, w_t, wt) of _prox_rows.  backward: proxtv_prox_fibers_vjp_dev_* -- gx = segment means of the upstream
        gradient, gw per edge."""
        @staticmethod
        def forward(ctx, x, w, w_t, wt):
            y = _prox_rows(x, w, wt)
            ctx.save_for_backward(y, wt)
            ctx.w = w
            ctx.w_like = (w_t.dtype, w_t.device, ()) if w_t is not None else None
            return y

        @staticmethod
        @once_differentiable
        def backward(ctx, gy):
            y, wt = ctx.saved_tensors
            need_x, _, need_w_t, need_wt = ctx.needs_input_grad
            B, L = y.shape
            g = gy.to(dtype=y.dtype).contiguous()
            gx = torch.empty_like(y)
            gw = torch.empty((B, max(L - 1, 0)), dtype=y.dtype, device=y.device) if (need_w_t or need_wt) else None
            _dev_call("prox_fibers_vjp_dev", y, y, g, gx, gw, B, L, 1, ctx.w, wt)
            g_w = _penalty_grad(gw, ctx.w_like) if need_w_t else None
            return (gx if need_x else None), None, g_w, (gw if need_wt else None)

    class TV2(torch.autograd.Function):
        """apply(xin, W1, W2, w, w_t, entry, geom) of _tv2_solve (W1 None: the penalty w, read from w_t when that is a tensor).
        backward: proxtv_<entry>_vjp_dev_* -- the exact vector-Jacobian product of the unrolled splitting (DR2_TV, DR2L1W_TV) or the
        Jacobian of the converged prox at the recorded partition (CP2_TV, CP2W_TV) -- with per-edge weight gradients (NULL for a map that
        needs none) or glam per image and axis; the upstream gradient is taken in the output's layout, the gradients come in their
        inputs'."""
        @staticmethod
        def forward(ctx, xin, W1, W2, w, w_t, entry, geom):
            M, N, batch, _, _, max_iters = geom
            tape_bytes, dr = _TAPED[entry]
            tape = torch.empty(int(tape_bytes(require_device(), M, N, batch, max_iters)), dtype=torch.uint8, device=xin.device)
            out = _tv2_solve(entry, xin, W1, W2, w, geom, tape)
            ctx.save_for_backward(tape, None if dr else out)
            ctx.entry, ctx.geom = entry, geom
            ctx.layouts = [(t.shape, t.stride(), t.dtype) if t is not None else None for t in (out, W1, W2)]
            ctx.w_like = (w_t.dtype, w_t.device, ()) if w_t is not None else None
            return out

        @staticmethod
        @once_differentiable
        def backward(ctx, gout):
            tape, out = ctx.saved_tensors
            M, N, batch, row_major, _, max_iters = ctx.geom
            dr = _TAPED[ctx.entry][1]
            need_x, need_w1, need_w2, _, need_w_t, _, _ = ctx.needs_input_grad

            def like(i):
                shape, stride, dt = ctx.layouts[i]
                return torch.empty_strided(shape, stride, dtype=dt, device=tape.device)
            g = like(0)                                   # the upstream gradient in the output's layout
            g.copy_(gout)
            gY = like(0)
            lead = (max_iters, tape) if dr else (tape, out)
            if ctx.layouts[1] is not None:
                gW1 = like(1) if need_w1 else None
                gW2 = like(2) if need_w2 else None
                _dev_call(ctx.entry + "_vjp_dev", g, M, N, batch, row_major, *lead, g, gY, gW1, gW2, *(() if dr else (None,)))
                return (gY if need_x else None), gW1, gW2, None, None, None, None
            glam = torch.empty(2 * batch, dtype=torch.float64, device=tape.device) if need_w_t else None
            _dev_call(ctx.entry + "_vjp_dev", g, M, N, batch, row_major, *lead, g, gY, glam)
            g_w = _penalty_grad(glam, ctx.w_like) if need_w_t else None
            return (gY if need_x else None), None, None, None, g_w, None, None

    class ND(torch.autograd.Function):
        """apply(xin, ws_t, solver, nsa, dsa, lama, max_iters, owner, batch, items) of _nd_solve; ctx also keeps the iteration count the
        solve ran (the Dykstra solvers' stop rule picks it; batch >= 1: each item's K).  backward: proxtv_<solver>_vjp_dev_*; the gradient
        of ws_t is npen * glam for PDR_TV and PD_TV (glam: the gradients of the scaled penalties), glam for PD2_TV.  batch >= 1:
        proxtv_<solver>_batched_vjp_dev_*, whose per-item glam is of the penalties as given for both solvers: summed over the items for a
        shared ws_t, the (batch, npen) rows themselves for a per-item one (items)."""
        @staticmethod
        def forward(ctx, xin, ws_t, solver, nsa, dsa, lama, max_iters, owner, batch, items=False):
            lib = require_device()
            if batch:
                tape_bytes = getattr(lib, "proxtv_%s_batched_tape_bytes" % solver)
                nb = int(tape_bytes(_ptr(nsa), len(nsa), len(dsa), batch, max_iters))
            else:
                tape_bytes = getattr(lib, "proxtv_%s_tape_bytes" % solver)
                nb = int(tape_bytes(_ptr(nsa), len(nsa), len(dsa), max_iters))  # 0: too large; the record call refuses it
            tape = torch.empty(max(nb, 256), dtype=torch.uint8, device=xin.device)
            out, info = _nd_solve(xin, solver, nsa, dsa, lama, max_iters, owner, batch, items, tape)
            ctx.save_for_backward(tape)
            iters = info[:, 0].astype(np.int64) if batch else int(info[0])
            ctx.geom, ctx.layout = (solver, nsa, dsa, max_iters, iters, batch, items), (out.shape, out.stride(), out.dtype)
            ctx.ws_like = (ws_t.dtype, ws_t.device, ws_t.shape) if ws_t is not None else None
            return out

        @staticmethod
        @once_differentiable
        def backward(ctx, gout):
            (tape,) = ctx.saved_tensors
            solver, nsa, dsa, max_iters, iters, batch, items = ctx.geom
            shape, stride, dt = ctx.layout
            need_x, need_ws = ctx.needs_input_grad[:2]
            npen = len(dsa)
            g = torch.empty_strided(shape, stride, dtype=dt, device=tape.device)      # the upstream gradient in the output's layout
            g.copy_(gout)
            gY = torch.empty_strided(shape, stride, dtype=dt, device=tape.device)
            glam = torch.empty(npen * max(batch, 1), dtype=torch.float64, device=tape.device) if need_ws else None
            rest = (None,) * (len(ctx.needs_input_grad) - 2)
            if batch:
                _dev_call(solver + "_batched_vjp_dev", g, nsa, len(nsa), npen, dsa, batch, max_iters, tape, g, gY, glam)
                g_ws = None
                if need_ws:
                    per_item = glam.view(batch, npen)
                    g_ws = _penalty_grad(per_item if items else per_item.sum(0, dtype=torch.float64), ctx.ws_like)
                return (gY if need_x else None), g_ws, *rest
            it = () if solver == "PDR_TV" else (iters,)                               # PDR_TV runs exactly max_iters iterations
            _dev_call(solver + "_vjp_dev", g, nsa, len(nsa), npen, dsa, max_iters, *it, tape, g, gY, glam)
            g_ws = _penalty_grad(glam if solver == "PD2_TV" else glam * float(npen), ctx.ws_like) if need_ws else None
            return (gY if need_x else None), g_ws, *rest

    return types.SimpleNamespace(ProxRows=ProxRows, TV2=TV2, ND=ND)
