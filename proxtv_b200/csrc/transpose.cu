// transpose.cu -- tiled gather/scatter between strided fibers and contiguous fibers.
//
// The fibers of a column-major array along a dimension d >= 1 have element stride inc = prod(ns[0..d-1]) and adjacent
// fibers are adjacent in memory: the array is [outer][len][inc] with `inc` fastest.  gather_fibers() writes the
// transposed slab [outer][inc][len] (every fiber contiguous), fusing the input op (A, A-B, A+B); scatter_fibers() is the
// inverse.  32 x 32 tiles through padded shared memory: both the read and the write side move 256-byte (f64) rows.
// This is the simple route for the strided direction while the scan itself is compute-bound; the tile kernel that stages
// strided fibers directly (DESIGN.md "next") removes these two extra sweeps.
#include "ptv_internal.h"
#include "chunk_core.cuh"
#include <stdint.h>

namespace ptv {

template <typename T>
__global__ void k_gather(const T* __restrict__ A, const T* __restrict__ B, int op, T* __restrict__ out, int len, long long inc,
                         int k_begin, int k_end) {
    __shared__ T tile[32][33];
    const long long o = blockIdx.z;
    const long long slab = (long long)len * inc;
    const long long r0 = (long long)blockIdx.x * 32;     // along inc (fiber index inside the slab)
    const int k0 = k_begin + blockIdx.y * 32;            // along the fiber (restricted to [k_begin, k_end))
    const int tx = threadIdx.x, ty = threadIdx.y;        // 32 x 8
    len = len < k_end ? len : k_end;
    const int flen = (int)(slab / inc);
    for (int dy = ty; dy < 32; dy += 8) {
        const int k = k0 + dy; const long long r = r0 + tx;
        if (k < len && r < inc) {
            const long long idx = o * slab + (long long)k * inc + r;
            T a = A[idx];
            if (op == IN_A_MINUS_B) a = a - B[idx]; else if (op == IN_A_PLUS_B) a = a + B[idx];
            tile[dy][tx] = a;
        }
    }
    __syncthreads();
    for (int dy = ty; dy < 32; dy += 8) {
        const long long r = r0 + dy; const int k = k0 + tx;
        if (k < len && r < inc) out[o * slab + r * flen + k] = tile[tx][dy];
    }
}

template <typename T>
__global__ void k_scatter(const T* __restrict__ in, T* __restrict__ X, int len, long long inc) {
    __shared__ T tile[32][33];
    const long long o = blockIdx.z;
    const long long slab = (long long)len * inc;
    const long long r0 = (long long)blockIdx.x * 32;
    const int k0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    for (int dy = ty; dy < 32; dy += 8) {
        const long long r = r0 + dy; const int k = k0 + tx;
        if (k < len && r < inc) tile[dy][tx] = in[o * slab + r * len + k];
    }
    __syncthreads();
    for (int dy = ty; dy < 32; dy += 8) {
        const int k = k0 + dy; const long long r = r0 + tx;
        if (k < len && r < inc) X[o * slab + (long long)k * inc + r] = tile[tx][dy];
    }
}

// scatter with a fused output form: X[g] = apply_out_ex(out_op, in(g), x(g)) where in(g) = A[g] (op) B[g] is recomputed exactly as
// the gather computed it, and x is the prox value coming back from the transposed layout.
// WOPS: also knows the weighted Douglas-Rachford forms (kept out of the default instance: the wider switch slows it measurably)
template <typename T, bool WOPS, bool EXPAND>
__global__ void k_scatter_ex(const T* __restrict__ in, const T* __restrict__ A, const T* __restrict__ B, const T* __restrict__ C, int op,
                             int out_op, T* __restrict__ X, int len, long long inc, long long r_begin, long long r_end,
                             const uint32_t* __restrict__ Mk, const T* __restrict__ Cv) {
    __shared__ T tile[32][33];
    __shared__ uint32_t pm[32];
    __shared__ T cvs[32];
    const long long o = blockIdx.z;
    const long long slab = (long long)len * inc;
    const long long r0 = r_begin + (long long)blockIdx.x * 32;
    const int k0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const long long rlim = inc < r_end ? inc : r_end;
    for (int dy = ty; dy < 32; dy += 8) {
        const long long r = r0 + dy; const int k = k0 + tx;
        if (k < len && r < rlim) tile[dy][tx] = in[o * slab + r * len + k];
    }
    if (EXPAND && ty == 0) {
        // sparse input (prox_fibers_chunked_contig_sparse): this tile is chunk k0/32 of 32 fibers; fetch their start masks and
        // entering values, the segment values themselves sit in the tile at their start positions
        const long long r = r0 + tx;
        if (r < rlim) { const long long e = (o * inc + r) * (long long)((len + 31) >> 5) + (k0 >> 5); pm[tx] = Mk[e]; cvs[tx] = Cv[e]; }
    }
    __syncthreads();
    for (int dy = ty; dy < 32; dy += 8) {
        const int k = k0 + dy; const long long r = r0 + tx;
        if (k < len && r < rlim) {
            const long long g = o * slab + (long long)k * inc + r;
            T yin = T(0);
            if (A) { yin = A[g]; if (op == IN_A_MINUS_B) yin = yin - B[g]; else if (op == IN_A_PLUS_B) yin = yin + B[g]; }   // A == nullptr: plain OUT_X
            T xv;
            if (EXPAND) { const uint32_t w = pm[tx] & (0xffffffffu >> (31 - dy)); xv = w ? tile[tx][high_bit(w)] : cvs[tx]; }
            else xv = tile[tx][dy];
            X[g] = WOPS ? apply_out_any<T>(out_op, yin, xv, A, B, C, g) : apply_out_ex<T>(out_op, yin, xv, A, B, C, g);
        }
    }
}

// ---- 64 x 64 tiles with 8-byte accesses for 4-byte element types: a 32 x 32 tile of floats moves only 128-byte rows and
//      leaves half of the memory pipeline idle.
//      Requirements (checked by the launchers): len, inc, k_begin/k_end, r_begin/r_end even and all bases 8-byte aligned. ----
struct alignas(8) F2 { float a, b; };
__device__ __forceinline__ float in_apply(int op, float a, float b) { return op == IN_A_MINUS_B ? a - b : (op == IN_A_PLUS_B ? a + b : a); }

__global__ void __launch_bounds__(256) k_gather_w(const float* __restrict__ A, const float* __restrict__ B, int op, float* __restrict__ out, int len,
                                                 long long inc, int k_begin, int k_end) {
    __shared__ float tile[64][65];
    const long long o = blockIdx.z, slab = (long long)len * inc;
    const long long r0 = (long long)blockIdx.x * 64;
    const int k0 = k_begin + blockIdx.y * 64;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int flen = len;
    len = len < k_end ? len : k_end;
    for (int dy = ty; dy < 64; dy += 8) {
        const int k = k0 + dy; const long long r = r0 + 2 * tx;
        if (k < len && r < inc) {
            const long long idx = o * slab + (long long)k * inc + r;
            F2 a = *reinterpret_cast<const F2*>(A + idx), b{0.f, 0.f};
            if (op != IN_A) b = *reinterpret_cast<const F2*>(B + idx);
            tile[dy][2 * tx] = in_apply(op, a.a, b.a); tile[dy][2 * tx + 1] = in_apply(op, a.b, b.b);
        }
    }
    __syncthreads();
    for (int dy = ty; dy < 64; dy += 8) {
        const long long r = r0 + dy; const int k = k0 + 2 * tx;
        if (k < len && r < inc) *reinterpret_cast<F2*>(out + o * slab + r * flen + k) = F2{tile[2 * tx][dy], tile[2 * tx + 1][dy]};
    }
}

template <bool WOPS, bool EX, bool EXPAND>
__global__ void __launch_bounds__(256) k_scatter_w(const float* __restrict__ in, const float* __restrict__ A, const float* __restrict__ B,
                                                  const float* __restrict__ C, int op, int out_op, float* __restrict__ X, int len, long long inc,
                                                  long long r_begin, long long r_end, const uint32_t* __restrict__ Mk, const float* __restrict__ Cv) {
    __shared__ float tile[64][65];
    __shared__ uint32_t pm[64][2];
    __shared__ float cvs[64][2];
    const long long o = blockIdx.z, slab = (long long)len * inc;
    const long long r0 = r_begin + (long long)blockIdx.x * 64;
    const int k0 = blockIdx.y * 64;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const long long rlim = inc < r_end ? inc : r_end;
    for (int dy = ty; dy < 64; dy += 8) {
        const long long r = r0 + dy; const int k = k0 + 2 * tx;
        if (k < len && r < rlim) { const F2 v = *reinterpret_cast<const F2*>(in + o * slab + r * len + k); tile[dy][2 * tx] = v.a; tile[dy][2 * tx + 1] = v.b; }
    }
    if (EXPAND && ty < 4) {                    // sparse input: start masks / entering values of the two chunks each tile row covers
        const int e = ty * 32 + tx, row = e >> 1, h = e & 1;
        const long long r = r0 + row;
        if (r < rlim && k0 + 32 * h < len) {
            const long long q = (o * inc + r) * (long long)((len + 31) >> 5) + (k0 >> 5) + h;
            pm[row][h] = Mk[q]; cvs[row][h] = Cv[q];
        }
    }
    __syncthreads();
    for (int dy = ty; dy < 64; dy += 8) {
        const int k = k0 + dy; const long long r = r0 + 2 * tx;
        if (k < len && r < rlim) {
            const long long g = o * slab + (long long)k * inc + r;
            F2 res;
            if (EXPAND) {
                const int h = dy >> 5; const uint32_t below = 0xffffffffu >> (31 - (dy & 31));
                const uint32_t w0 = pm[2 * tx][h] & below, w1 = pm[2 * tx + 1][h] & below;
                res.a = w0 ? tile[2 * tx][32 * h + high_bit(w0)] : cvs[2 * tx][h];
                res.b = w1 ? tile[2 * tx + 1][32 * h + high_bit(w1)] : cvs[2 * tx + 1][h];
            } else res = F2{tile[2 * tx][dy], tile[2 * tx + 1][dy]};
            if (EX) {
                const F2 a = *reinterpret_cast<const F2*>(A + g);
                F2 b{0.f, 0.f};
                if (op != IN_A) b = *reinterpret_cast<const F2*>(B + g);
                const float y0 = in_apply(op, a.a, b.a), y1 = in_apply(op, a.b, b.b);
                res.a = WOPS ? apply_out_any<float>(out_op, y0, res.a, A, B, C, g) : apply_out_ex<float>(out_op, y0, res.a, A, B, C, g);
                res.b = WOPS ? apply_out_any<float>(out_op, y1, res.b, A, B, C, g + 1) : apply_out_ex<float>(out_op, y1, res.b, A, B, C, g + 1);
            }
            *reinterpret_cast<F2*>(X + g) = res;
        }
    }
}
static inline bool wide_ok(const void* a, const void* b, const void* c, const void* d, const void* e, long long len, long long inc,
                           long long lo, long long hi) {
    const uintptr_t m = (uintptr_t)a | (uintptr_t)b | (uintptr_t)c | (uintptr_t)d | (uintptr_t)e;
    return (m & 7) == 0 && len % 2 == 0 && inc % 2 == 0 && lo % 2 == 0 && hi % 2 == 0;
}
// float front ends: the wide kernels when the shape allows, else fall through (return false) to the generic 32 x 32 tiles
static bool gather_wide(const float* A, const float* B, int op, float* out, int len, long long inc, int k_begin, int k_end, unsigned gz,
                        cudaStream_t st) {
    if (!wide_ok(A, B, out, nullptr, nullptr, len, inc, k_begin, k_end)) return false;
    dim3 grid((unsigned)((inc + 63) / 64), (unsigned)((k_end - k_begin + 63) / 64), gz), block(32, 8);
    k_gather_w<<<grid, block, 0, st>>>(A, B, op, out, len, inc, k_begin, k_end);
    return true;
}
static bool gather_wide(const double*, const double*, int, double*, int, long long, int, int, unsigned, cudaStream_t) { return false; }
static bool scatter_wide(const float* in, const float* A, const float* B, const float* C, int op, int out_op, bool ex, float* X, int len,
                         long long inc, long long r_begin, long long r_end, unsigned gz, cudaStream_t st, const uint32_t* Mk = nullptr,
                         const float* Cv = nullptr) {
    if (!wide_ok(in, A, B, C, X, len, inc, r_begin, r_end)) return false;
    dim3 grid((unsigned)((r_end - r_begin + 63) / 64), (unsigned)((len + 63) / 64), gz), block(32, 8);
    if (Mk) {
        if (!ex) k_scatter_w<false, false, true><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, Mk, Cv);
        else if (out_op >= OUT_DRW_ROWS) k_scatter_w<true, true, true><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, Mk, Cv);
        else k_scatter_w<false, true, true><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, Mk, Cv);
    } else {
        if (!ex) k_scatter_w<false, false, false><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, nullptr, nullptr);
        else if (out_op >= OUT_DRW_ROWS) k_scatter_w<true, true, false><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, nullptr, nullptr);
        else k_scatter_w<false, true, false><<<grid, block, 0, st>>>(in, A, B, C, op, out_op, X, len, inc, r_begin, r_end, nullptr, nullptr);
    }
    return true;
}
static bool scatter_wide(const double*, const double*, const double*, const double*, int, int, bool, double*, int, long long, long long,
                         long long, unsigned, cudaStream_t, const uint32_t* = nullptr, const double* = nullptr) { return false; }

template <typename T>
cudaError_t scatter_fibers_ex(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g, cudaStream_t st) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    const long long outer = g.nf / g.inc;
    dim3 grid((unsigned)((g.inc + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    for (long long o0 = 0; o0 < outer; o0 += 65535) {
        grid.z = (unsigned)((outer - o0) < 65535 ? (outer - o0) : 65535);
        const long long off = o0 * (long long)g.len * g.inc;
        if (scatter_wide(in + off, A + off, B ? B + off : nullptr, C ? C + off : nullptr, (int)op, out_op, true, X + off, g.len, g.inc, 0, g.inc, grid.z, st)) continue;
        if (out_op >= OUT_DRW_ROWS)
            k_scatter_ex<T, true, false><<<grid, block, 0, st>>>(in + off, A + off, B ? B + off : nullptr, C ? C + off : nullptr, (int)op, out_op, X + off, g.len, g.inc, 0, g.inc, nullptr, nullptr);
        else
            k_scatter_ex<T, false, false><<<grid, block, 0, st>>>(in + off, A + off, B ? B + off : nullptr, C ? C + off : nullptr, (int)op, out_op, X + off, g.len, g.inc, 0, g.inc, nullptr, nullptr);
    }
    return cudaGetLastError();
}
template cudaError_t scatter_fibers_ex<double>(const double*, const double*, const double*, const double*, InOp, int, double*, FiberGeom, cudaStream_t);
template cudaError_t scatter_fibers_ex<float>(const float*, const float*, const float*, const float*, InOp, int, float*, FiberGeom, cudaStream_t);

template <typename T>
cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    const long long outer = g.nf / g.inc;
    dim3 grid((unsigned)((g.inc + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    for (long long o0 = 0; o0 < outer; o0 += 65535) {                // gridDim.z limit
        grid.z = (unsigned)((outer - o0) < 65535 ? (outer - o0) : 65535);
        const long long off = o0 * (long long)g.len * g.inc;
        if (gather_wide(A + off, B ? B + off : nullptr, (int)op, out + off, g.len, g.inc, 0, g.len, grid.z, st)) continue;
        k_gather<T><<<grid, block, 0, st>>>(A + off, B ? B + off : nullptr, (int)op, out + off, g.len, g.inc, 0, g.len);
    }
    return cudaGetLastError();
}
template <typename T>
cudaError_t scatter_fibers(const T* in, T* X, FiberGeom g, cudaStream_t st) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    const long long outer = g.nf / g.inc;
    dim3 grid((unsigned)((g.inc + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    for (long long o0 = 0; o0 < outer; o0 += 65535) {
        grid.z = (unsigned)((outer - o0) < 65535 ? (outer - o0) : 65535);
        const long long off = o0 * (long long)g.len * g.inc;
        if (scatter_wide(in + off, nullptr, nullptr, nullptr, 0, 0, false, X + off, g.len, g.inc, 0, g.inc, grid.z, st)) continue;
        k_scatter<T><<<grid, block, 0, st>>>(in + off, X + off, g.len, g.inc);
    }
    return cudaGetLastError();
}

// sub-range forms for the pipelined Douglas-Rachford driver (single slab: g.nf == g.inc)
template <typename T>
cudaError_t gather_fibers_range(const T* A, const T* B, InOp op, T* out, FiberGeom g, int k_begin, int k_end, cudaStream_t st) {
    if (k_end <= k_begin) return cudaSuccess;
    if (gather_wide(A, B, (int)op, out, g.len, g.inc, k_begin, k_end, 1, st)) return cudaGetLastError();
    dim3 grid((unsigned)((g.inc + 31) / 32), (unsigned)((k_end - k_begin + 31) / 32), 1), block(32, 8);
    k_gather<T><<<grid, block, 0, st>>>(A, B, (int)op, out, g.len, g.inc, k_begin, k_end);
    return cudaGetLastError();
}
template <typename T>
cudaError_t scatter_fibers_ex_range(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g,
                                    long long r_begin, long long r_end, cudaStream_t st) {
    if (r_end <= r_begin) return cudaSuccess;
    if (scatter_wide(in, A, B, C, (int)op, out_op, true, X, g.len, g.inc, r_begin, r_end, 1, st)) return cudaGetLastError();
    dim3 grid((unsigned)((r_end - r_begin + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    if (out_op >= OUT_DRW_ROWS) k_scatter_ex<T, true, false><<<grid, block, 0, st>>>(in, A, B, C, (int)op, out_op, X, g.len, g.inc, r_begin, r_end, nullptr, nullptr);
    else k_scatter_ex<T, false, false><<<grid, block, 0, st>>>(in, A, B, C, (int)op, out_op, X, g.len, g.inc, r_begin, r_end, nullptr, nullptr);
    return cudaGetLastError();
}
// fused scatter of a SPARSE prox result (see prox_fibers_chunked_contig_sparse): expands the segments while it transposes
template <typename T>
cudaError_t scatter_fibers_ex_sparse_range(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op,
                                           T* X, FiberGeom g, long long r_begin, long long r_end, cudaStream_t st) {
    if (r_end <= r_begin) return cudaSuccess;
    if (scatter_wide(in, A, B, C, (int)op, out_op, true, X, g.len, g.inc, r_begin, r_end, 1, st, Mk, Cv)) return cudaGetLastError();
    dim3 grid((unsigned)((r_end - r_begin + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    if (out_op >= OUT_DRW_ROWS) k_scatter_ex<T, true, true><<<grid, block, 0, st>>>(in, A, B, C, (int)op, out_op, X, g.len, g.inc, r_begin, r_end, Mk, Cv);
    else k_scatter_ex<T, false, true><<<grid, block, 0, st>>>(in, A, B, C, (int)op, out_op, X, g.len, g.inc, r_begin, r_end, Mk, Cv);
    return cudaGetLastError();
}
// whole-geometry form (any number of slabs).  A == nullptr: plain scatter of the expanded prox values (IN_A / OUT_X semantics).
template <typename T>
cudaError_t scatter_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                  FiberGeom g, cudaStream_t st) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    const long long outer = g.nf / g.inc, lpf = ((long long)g.len + 31) / 32;
    const bool ex = A != nullptr;
    dim3 grid((unsigned)((g.inc + 31) / 32), (unsigned)((g.len + 31) / 32), 1), block(32, 8);
    for (long long o0 = 0; o0 < outer; o0 += 65535) {
        grid.z = (unsigned)((outer - o0) < 65535 ? (outer - o0) : 65535);
        const long long off = o0 * (long long)g.len * g.inc, moff = o0 * g.inc * lpf;
        const T* Ao = ex ? A + off : nullptr;          // plain form: OUT_X never looks at the input
        if (scatter_wide(in + off, Ao, (ex && B) ? B + off : nullptr, (ex && C) ? C + off : nullptr, ex ? (int)op : (int)IN_A, ex ? out_op : (int)OUT_X,
                         ex, X + off, g.len, g.inc, 0, g.inc, grid.z, st, Mk + moff, Cv + moff)) continue;
        if (ex && out_op >= OUT_DRW_ROWS)
            k_scatter_ex<T, true, true><<<grid, block, 0, st>>>(in + off, Ao, B ? B + off : nullptr, C ? C + off : nullptr, (int)op, out_op, X + off, g.len, g.inc, 0, g.inc, Mk + moff, Cv + moff);
        else
            k_scatter_ex<T, false, true><<<grid, block, 0, st>>>(in + off, Ao, (ex && B) ? B + off : nullptr, (ex && C) ? C + off : nullptr, ex ? (int)op : (int)IN_A,
                                                                 ex ? out_op : (int)OUT_X, X + off, g.len, g.inc, 0, g.inc, Mk + moff, Cv + moff);
    }
    return cudaGetLastError();
}
// Expand a SPARSE prox result over CONTIGUOUS fibers g (prox_fibers_chunked_contig_sparse) with a fused output form, in the fibers'
// own layout: X[e] = apply_out_any(out_op, A[e] (op) B[e], x, A, B, C, e), x the value of the segment that covers e.  The chunked
// kernel's fill only knows the forms of apply_out_ex (the weighted Douglas-Rachford ones would fatten its loop for every caller), so
// the contiguous row pass of C-ordered weighted images ends here instead.  One warp per 32-sample window: its start mask and
// entering value are one broadcast load each, the segment values lie in the window itself.  X may not alias in.
template <typename T>
__global__ void __launch_bounds__(256) k_expand_sparse(const T* __restrict__ in, const uint32_t* __restrict__ Mk, const T* __restrict__ Cv,
                                                       const T* A, const T* B, const T* C, int op, int out_op, T* X, long long nf, int len) {
    const int lane = threadIdx.x & 31;
    const long long lpf = ((long long)len + 31) >> 5, nw = nf * lpf;
    const uint32_t below = 0xffffffffu >> (31 - lane);
    for (long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nw; q += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long f = q / lpf, c = q - f * lpf;
        const uint32_t m = Mk[q] & below;
        const T cv = Cv[q];
        const long long w0 = f * len + c * 32, k = c * 32 + lane;
        if (k < len) {
            const long long e = w0 + lane;
            const T xv = m ? in[w0 + high_bit(m)] : cv;
            T yin = A[e];
            if (op == IN_A_MINUS_B) yin = yin - B[e]; else if (op == IN_A_PLUS_B) yin = yin + B[e];
            X[e] = apply_out_any<T>(out_op, yin, xv, A, B, C, e);
        }
    }
}
template <typename T>
cudaError_t expand_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                 FiberGeom g, cudaStream_t st) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    if (g.inc != 1) return cudaErrorInvalidValue;
    const long long warps = g.nf * (((long long)g.len + 31) / 32);
    long long blocks = (warps + 7) / 8;
    if (blocks > 132LL * 16) blocks = 132LL * 16;
    k_expand_sparse<T><<<(unsigned)blocks, 256, 0, st>>>(in, Mk, Cv, A, B, C, (int)op, out_op, X, g.nf, g.len);
    return cudaGetLastError();
}

#define INST_R(T) \
    template cudaError_t expand_fibers_sparse<T>(const T*, const uint32_t*, const T*, const T*, const T*, const T*, InOp, int, T*, FiberGeom, cudaStream_t); \
    template cudaError_t scatter_fibers_sparse<T>(const T*, const uint32_t*, const T*, const T*, const T*, const T*, InOp, int, T*, FiberGeom, cudaStream_t); \
    template cudaError_t scatter_fibers_ex_sparse_range<T>(const T*, const uint32_t*, const T*, const T*, const T*, const T*, InOp, int, T*, FiberGeom, long long, long long, cudaStream_t); \
    template cudaError_t gather_fibers_range<T>(const T*, const T*, InOp, T*, FiberGeom, int, int, cudaStream_t); \
    template cudaError_t scatter_fibers_ex_range<T>(const T*, const T*, const T*, const T*, InOp, int, T*, FiberGeom, long long, long long, cudaStream_t);
INST_R(double)
INST_R(float)

template cudaError_t gather_fibers<double>(const double*, const double*, InOp, double*, FiberGeom, cudaStream_t);
template cudaError_t gather_fibers<float>(const float*, const float*, InOp, float*, FiberGeom, cudaStream_t);
template cudaError_t scatter_fibers<double>(const double*, double*, FiberGeom, cudaStream_t);
template cudaError_t scatter_fibers<float>(const float*, float*, FiberGeom, cudaStream_t);

}  // namespace ptv
