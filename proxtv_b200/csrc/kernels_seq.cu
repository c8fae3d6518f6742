// kernels_seq.cu -- robust baseline: one lane runs the whole sequential scan of one fiber.
//
// Works for any fiber length, stride and weight; used for tiny problems, as the repair path for fibers the chunked
// kernels flag, and as the on-device cross-check of the fast kernels.  With adjacent lanes on adjacent fibers the
// strided direction (inc > 1) is naturally coalesced; contiguous fibers rely on L1 (each lane streams its own lines).
// Reference behaviour: TV() with p == 1 applied to each fiber (src/TVgenopt.cpp:41-47, src/TVNDopt.cpp:182-207).
#include "ptv_internal.h"
#include "chunk_core.cuh"

namespace ptv {

// LAMF: fiber j's penalty is lamf[j / fpi] (one per group of fpi fibers), the uniform scan with that value
template <typename T, bool WEIGHTED, bool LAMF = false>
__global__ void __launch_bounds__(32) k_prox_seq(const T* __restrict__ A, const T* __restrict__ B, const T* __restrict__ C, int op, T* __restrict__ X,
                                                 int out_op, FiberGeom g, T lam, const T* __restrict__ lamv,
                                                 const int* __restrict__ list, long long nlist, const T* __restrict__ lamf, long long fpi) {
    long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (list) { if (j >= nlist) return; j = list[j]; }
    else if (j >= g.nf) return;
    const int n = g.len;
    const long long inc = g.inc;
    const long long base = (j / inc) * inc * n + (j % inc);
    const long long wbase = (j / inc) * inc * (n - 1) + (j % inc);
    auto y = [&](int i) -> T {
        long long o = base + (long long)i * inc;
        T a = A[o];
        return op == IN_A ? a : (op == IN_A_MINUS_B ? a - B[o] : a + B[o]);
    };
    auto run = [&](auto lamf) {
        Scan<T> s;
        s.begin(0, y, lamf);
        int f, l; T v;
        while (s.i < n) {
            int k = s.step(n, y, lamf, f, l, v);
            if (k != K_NONE)
                for (int q = f; q <= l; q++) { const long long g2 = base + (long long)q * inc; X[g2] = out_op ? apply_out_any<T>(out_op, y(q), v, A, B, C, g2) : v; }
        }
        for (int q = s.last + 1; q < n; q++) { const long long g2 = base + (long long)q * inc; X[g2] = out_op ? apply_out_any<T>(out_op, y(q), s.lo, A, B, C, g2) : s.lo; }
    };
    if (n <= 0) return;
    if (WEIGHTED) {
        if (n == 1) { X[base] = apply_out_any<T>(out_op, y(0), y(0), A, B, C, base); return; }     // the reference reads lambda[0] out of bounds here; identity is the limit
        auto ld = [&](int i) -> T { return lamv[wbase + (long long)i * inc]; };
        run(ArrayLam<T, decltype(ld)>{ld});
    } else {
        run(UniformLam<T>{LAMF ? lamf[j / fpi] : lam});
    }
}

// prox of a CONSTANT fiber (all samples equal c[b]) of length n, one thread per fiber, everything in registers.
// Used for the first Douglas-Rachford pass, whose input is the constant image 2*mean (src/TV2Dopt.cpp:390-395): all fibers
// of an image are then identical, so one fiber per image is solved and broadcast.  x1: [batch][n].
template <typename T>
__global__ void k_prox_const_fiber(const T* __restrict__ c, long long c_stride, int n, T lam, T* __restrict__ x1) {
    const long long b = blockIdx.x;
    const T cv = c[b * c_stride];
    auto y = [cv](int) -> T { return cv; };
    UniformLam<T> lamf{lam};
    T* out = x1 + b * (long long)n;
    Scan<T> s;
    s.begin(0, y, lamf);
    int f, l; T v;
    while (s.i < n) {
        const int i = s.i, d = i - s.last;
        if (i < n - 1 && d < 65536) {
            // regular step with the division a/d done as a*r + Markstein correction (== IEEE a/d, see chunk_core.cuh); the
            // reciprocal r = 1/d only depends on the loop counters, so its (IEEE) division is off the dependent chain --
            // a constant fiber never breaks, d runs up to n, and two chained IEEE divisions per step were the whole cost.
            const T dd = T(d), r = T(1) / dd;
            const T hlo = s.hlo + (s.lo - cv), hhi = s.hhi + (s.hi - cv);
            if (!(lam < hlo) && !(-lam > hhi)) {
                const T nh = lam - hhi, nl = -lam - hlo;
                const T qh0 = nh * r, ql0 = nl * r;
                const T qh = fma(fma(-qh0, dd, nh), r, qh0), ql = fma(fma(-ql0, dd, nl), r, ql0);
                const bool thi = hhi >= lam, tlo = hlo <= -lam;
                s.hi = thi ? s.hi + qh : s.hi;  s.hhi = thi ? lam : hhi;   s.bhi = thi ? i : s.bhi;
                s.lo = tlo ? s.lo + ql : s.lo;  s.hlo = tlo ? -lam : hlo;  s.blo = tlo ? i : s.blo;
                s.i = i + 1;
                continue;
            }
        }
        int k = s.step(n, y, lamf, f, l, v);          // breaks (none expected on a constant fiber) and the closing sample
        if (k != K_NONE) for (int q = f; q <= l; q++) out[q] = v;
    }
    for (int q = s.last + 1; q < n; q++) out[q] = s.lo;
}
template <typename T>
cudaError_t prox_const_fibers(const T* c, long long c_stride, int batch, int n, T lam, T* x1, cudaStream_t st) {
    if (batch <= 0 || n <= 0) return cudaSuccess;
    k_prox_const_fiber<T><<<batch, 1, 0, st>>>(c, c_stride, n, lam, x1);
    return cudaGetLastError();
}
template cudaError_t prox_const_fibers<double>(const double*, long long, int, int, double, double*, cudaStream_t);
template cudaError_t prox_const_fibers<float>(const float*, long long, int, int, float, float*, cudaStream_t);

template <typename T>
cudaError_t prox_fibers_seq(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv,
                            const int* list, long long nlist, cudaStream_t st, const T* lamf, long long fpi) {
    long long cnt = list ? nlist : g.nf;
    if (cnt <= 0 || g.len <= 0) return cudaSuccess;
    unsigned blocks = (unsigned)((cnt + 31) / 32);
    if (lamv) k_prox_seq<T, true><<<blocks, 32, 0, st>>>(A, B, C, (int)op, X, out_op, g, lam, lamv, list, nlist, nullptr, 1);
    else if (lamf) k_prox_seq<T, false, true><<<blocks, 32, 0, st>>>(A, B, C, (int)op, X, out_op, g, lam, nullptr, list, nlist, lamf, fpi);
    else      k_prox_seq<T, false><<<blocks, 32, 0, st>>>(A, B, C, (int)op, X, out_op, g, lam, lamv, list, nlist, nullptr, 1);
    return cudaGetLastError();
}

template cudaError_t prox_fibers_seq<double>(const double*, const double*, const double*, InOp, double*, int, FiberGeom, double, const double*,
                                             const int*, long long, cudaStream_t, const double*, long long);
template cudaError_t prox_fibers_seq<float>(const float*, const float*, const float*, InOp, float*, int, FiberGeom, float, const float*,
                                            const int*, long long, cudaStream_t, const float*, long long);

}  // namespace ptv
