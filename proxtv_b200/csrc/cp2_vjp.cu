// cp2_vjp.cu -- the backward pass of the converged 2D TV-L1 prox (CondatChambollePock2_TV alg 0 / 1 and its weighted form, DESIGN.md
// section 15.2): a fused-edge tape written after the recorded forward, and the vector-Jacobian product of the prox at that partition.
//
// Anisotropic TV-L1 makes y = prox(x) constant on clusters: connected sets of pixels joined by fused edges.  Away from ties the
// Jacobian with respect to x is the orthogonal projection onto functions constant on clusters, and for a cut edge e = (i, j) (j the
// successor of i along its axis) the derivative with respect to its weight is sgn(y_j - y_i) (gx_i - gx_j).  The contract, per image:
//   1. edge e = (i, j) is FUSED iff w_e > 0 and (|U_e| < w_e or y_i == y_j as stored), U_e the final dual of the iteration that produced
//      the result (clip() returns the bound itself when it clips, so |U_e| < w_e is exact in either dtype); a NaN never fuses;
//   2. clusters are the 4-connected components of the fused edges;
//   3. S_C = sum over C of (double) g_i, gx_i = (T)(S_C / |C|);
//   4. gw_e = (T)(sgn(y_j - y_i) ((double) gx_i - (double) gx_j)) on cut edges, +0 on fused ones; glam = per image [sum of gw along
//      axis 0, along axis 1] in double.
// S_C is computed exactly: every g_i is split into three 32-bit limbs of a 93-bit fixed-point value scaled to the cluster's largest
// exponent, the limbs are summed with integer atomics (whose result does not depend on their order), and the 96-bit total is rounded
// to double once.  Only parts below 2^-93 of the cluster's largest |g| are dropped.  So gx does not depend on timing or on the storage
// order.  glam is a two-stage double sum in a fixed order over the column-major (canonical) index, also the same in both orders.
//
// Tape: a 256-byte header (Cp2TapeHeader), then two bitsets in storage order of vjp_tape_set_bytes(n) bytes each (vjp_core.cuh
// layout): bit q of the first is "q is fused with its successor along the contiguous axis F", of the second "along the strided axis S".
//
// Labelling: union-find over the canonical (column-major) image-local index with atomic-min hooking, so every root is its cluster's
// smallest canonical index whatever order the unions take; then one flatten pass.  Labels are image-local int32 (M N < 2^31).
#include "ptv_internal.h"
#include "vjp_core.cuh"
#include <limits.h>
#include <string.h>

namespace ptv {

namespace {

struct Cp2TapeHeader {
    uint64_t magic;
    int64_t elem, M, N, batch, row_major, weighted;
    int64_t pad[25];
};
static_assert(sizeof(Cp2TapeHeader) == 256, "tape header is 256 bytes");
constexpr uint64_t CP2_TAPE_MAGIC = 0x3150415456325043ull;          // "CP2VTAP1"
constexpr int FIX_BITS = 93;                                          // fixed-point bits of one summand below its cluster's top exponent
constexpr int GLAM_CHUNK = 4096;                                      // canonical elements per first-stage glam block
constexpr int NO_EXP = (int)0x80808080;                               // the exponent slot's fill: no nonzero summand yet
constexpr int BAD_EXP = INT_MAX;                                      // a non-finite summand: the cluster's sum is NaN

inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
unsigned grid_for(long long n) { long long b = (n + 255) / 256; return (unsigned)(b < 1 ? 1 : (b > 132LL * 16 ? 132LL * 16 : b)); }

// image geometry in storage terms (F contiguous, S strided) and the canonical index c = i + M j of element (f, s)
struct G2 {
    int F, S, M, row_major;
    long long img, n;
    __device__ __forceinline__ int canon(int f, int s) const { return row_major ? s + S * f : f + F * s; }
};

#define GRID_STRIDE(q, n) for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < (n); q += (long long)gridDim.x * blockDim.x)

__device__ __forceinline__ bool tape_bit(const uint32_t* w, long long q) { return (w[q >> 5] >> (q & 31)) & 1u; }

// ---------------------------------------------------------------- tape (after the recorded forward)
// One warp per 32-element word.  The duals of image b are the buffer its last iteration wrote, ((st - 1) & 1) like k_cp2_out.
template <typename T, bool WTD>
__global__ void k_cp2_tape(G2 g, const T* __restrict__ X, const T* __restrict__ Uf0, const T* __restrict__ Uf1, const T* __restrict__ Us0,
                           const T* __restrict__ Us1, const int* __restrict__ stopped, int it_end, T lam, const T* __restrict__ Wf,
                           const T* __restrict__ Ws, uint32_t* __restrict__ BF, uint32_t* __restrict__ BS, long long nwords) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, wstep = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long wd = w0; wd < nwords; wd += wstep) {
        const long long q = wd * 32 + lane;
        bool ff = false, fs = false;
        if (q < g.n) {
            const long long b = q / g.img, e = q - b * g.img;
            const int f = (int)(e % g.F), s = (int)(e / g.F);
            const int st = stopped[b] ? stopped[b] : it_end;
            const bool odd = ((st - 1) & 1) != 0;
            const T x = X[q];
            if (f < g.F - 1) {
                const T w = WTD ? Wf[q - (b * g.S + s)] : lam, u = odd ? Uf1[q] : Uf0[q];
                ff = w > T(0) && (fabs(u) < w || x == X[q + 1]);
            }
            if (s < g.S - 1) {
                const T w = WTD ? Ws[q - b * g.F] : lam, u = odd ? Us1[q] : Us0[q];
                fs = w > T(0) && (fabs(u) < w || x == X[q + g.F]);
            }
        }
        const uint32_t bf = __ballot_sync(0xffffffffu, ff), bs = __ballot_sync(0xffffffffu, fs);
        if (lane == 0) { BF[wd] = bf; BS[wd] = bs; }
    }
}

// ---------------------------------------------------------------- connected components
// the root of c, halving the path on the way (each visited node is pointed at its grandparent: still an ancestor, so a racing union
// loses no link it depends on -- a hook that lands on a node that was no root is followed up by its caller)
__device__ __forceinline__ int cc_find(int* P, int c) {
    int p = __ldcg(P + c);
    if (p == c) return c;
    int prev = c, next;
    while (p > (next = __ldcg(P + p))) { __stcg(P + prev, next); prev = p; p = next; }
    return p;
}
// joins the trees of a and b: the larger root is hooked under the smaller with atomicMin; a root that was hooked meanwhile hands over
// to its new parent
__device__ void cc_unite(int* P, int a, int b) {
    for (;;) {
        a = cc_find(P, a); b = cc_find(P, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(P + a, b);
        if (old == a) return;
        a = old;
    }
}

__global__ void k_cc_init(G2 g, int* __restrict__ P) {
    GRID_STRIDE(q, g.n) P[q] = (int)(q % g.img);
}

__global__ void k_cc_union(G2 g, const uint32_t* __restrict__ BF, const uint32_t* __restrict__ BS, int* P) {
    GRID_STRIDE(q, g.n) {
        const bool ff = tape_bit(BF, q), fs = tape_bit(BS, q);
        if (!ff && !fs) continue;
        const long long b = q / g.img, e = q - b * g.img;
        const int f = (int)(e % g.F), s = (int)(e / g.F);
        int* Pb = P + b * g.img;
        const int c = g.canon(f, s);
        if (ff) cc_unite(Pb, c, g.canon(f + 1, s));
        if (fs) cc_unite(Pb, c, g.canon(f, s + 1));
    }
}

// Every store here is a root, so a walk that reads one only gets shorter; the walk must not halve paths itself: a halving store that
// lands after another thread's store of the root would leave a node pointing at a non-root.
__global__ void k_cc_flatten(G2 g, int* P) {
    GRID_STRIDE(q, g.n) {
        const int* Pb = P + (q / g.img) * g.img;
        int c = (int)(q % g.img), p = __ldcg(Pb + c);
        while (p != c) { c = p; p = __ldcg(Pb + c); }
        __stcg(P + q, c);
    }
}

// ---------------------------------------------------------------- exact cluster sums
// the root slot (b img + root) of storage element q
__device__ __forceinline__ long long root_slot(const G2& g, const int* P, long long q) {
    const long long b = q / g.img, e = q - b * g.img;
    return b * g.img + P[b * g.img + g.canon((int)(e % g.F), (int)(e / g.F))];
}

// A warp whose 32 elements share one root (the common case inside large clusters) adds once for all of them.
__device__ __forceinline__ bool warp_uniform(bool valid, long long R) {
    const long long R0 = __shfl_sync(0xffffffffu, R, 0);
    return __all_sync(0xffffffffu, valid && R == R0);
}

// count and largest binary exponent of each cluster's nonzero summands (BAD_EXP: a non-finite one)
template <typename T>
__global__ void k_sum_scale(G2 g, const int* __restrict__ P, const T* __restrict__ gin, int* cnt, int* emax) {
    for (long long base = ((long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31LL; base < g.n; base += (long long)gridDim.x * blockDim.x) {
        const long long q = base + (threadIdx.x & 31);
        const bool valid = q < g.n;
        long long R = 0; int e = NO_EXP;
        if (valid) {
            R = root_slot(g, P, q);
            const double v = (double)gin[q];
            if (!isfinite(v)) e = BAD_EXP;
            else if (v != 0.0) frexp(v, &e);
        }
        if (warp_uniform(valid, R)) {
            const int m = __reduce_max_sync(0xffffffffu, e);
            if ((threadIdx.x & 31) == 0) { atomicAdd(cnt + R, 32); if (m != NO_EXP) atomicMax(emax + R, m); }
        } else if (valid) {
            atomicAdd(cnt + R, 1);
            if (e != NO_EXP) atomicMax(emax + R, e);
        }
    }
}

// the three limbs of |v| 2^(FIX_BITS - E), truncated, with v's sign (|v| < 2^E)
__device__ __forceinline__ void limbs(double v, int E, long long l[3]) {
    const double a = ldexp(fabs(v), FIX_BITS - E);                    // exact: a power-of-two scaling into [0, 2^93)
    const double h = floor(ldexp(a, -64)), r = a - ldexp(h, 64);      // exact: r < 2^64 keeps the low bits of a
    const double m = floor(ldexp(r, -32)), lo = floor(r - ldexp(m, 32));
    const long long sg = v < 0 ? -1 : 1;
    l[0] = sg * (long long)lo; l[1] = sg * (long long)m; l[2] = sg * (long long)h;
}

template <typename T>
__global__ void k_sum_add(G2 g, const int* __restrict__ P, const T* __restrict__ gin, const int* __restrict__ emax, long long* acc) {
    for (long long base = ((long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31LL; base < g.n; base += (long long)gridDim.x * blockDim.x) {
        const long long q = base + (threadIdx.x & 31);
        const bool valid = q < g.n;
        long long R = 0, l[3] = {0, 0, 0};
        if (valid) {
            R = root_slot(g, P, q);
            const double v = (double)gin[q];
            const int E = emax[R];
            if (v != 0.0 && E != BAD_EXP) limbs(v, E, l);
        }
        if (warp_uniform(valid, R)) {
            for (int k = 0; k < 3; k++)
                for (int o = 16; o > 0; o >>= 1) l[k] += __shfl_down_sync(0xffffffffu, l[k], o);   // exact: 32 limbs < 2^37
            if ((threadIdx.x & 31) == 0)
                for (int k = 0; k < 3; k++) if (l[k]) atomicAdd((unsigned long long*)(acc + 3 * R + k), (unsigned long long)l[k]);
        } else if (valid) {
            for (int k = 0; k < 3; k++) if (l[k]) atomicAdd((unsigned long long*)(acc + 3 * R + k), (unsigned long long)l[k]);
        }
    }
}

// the cluster sum from its limbs: the 128-bit total (|total| < 2^124: 2^31 summands < 2^93) rounded to double once
__device__ __forceinline__ double cluster_sum(const long long* acc, int E) {
    if (E == BAD_EXP) return __longlong_as_double(0x7ff8000000000000LL);
    if (E == NO_EXP) return 0.0;
    const __int128 t = (__int128)acc[0] + ((__int128)acc[1] << 32) + ((__int128)acc[2] << 64);
    const bool neg = t < 0;
    const unsigned __int128 u = neg ? (unsigned __int128)(-t) : (unsigned __int128)t;
    const unsigned long long hi = (unsigned long long)(u >> 64);
    double d;
    if (hi == 0) {
        d = (double)(unsigned long long)u;                            // one rounding
    } else {
        const int sh = 64 - __clzll((long long)hi);                   // bits above the low 64
        unsigned long long top = (unsigned long long)(u >> sh);
        if ((unsigned long long)u & ((1ull << sh) - 1)) top |= 1ull;  // sticky: the bits shifted out decide a tie
        d = ldexp((double)top, sh);
    }
    return ldexp(neg ? -d : d, E - FIX_BITS);
}

template <typename T>
__global__ void k_gx(G2 g, const int* __restrict__ P, const int* __restrict__ cnt, const int* __restrict__ emax, const long long* __restrict__ acc,
                     T* __restrict__ gx) {
    GRID_STRIDE(q, g.n) {
        const long long R = root_slot(g, P, q);
        gx[q] = (T)(cluster_sum(acc + 3 * R, emax[R]) / (double)cnt[R]);
    }
}

// ---------------------------------------------------------------- edge gradients
template <typename T>
__device__ __forceinline__ double edge_gw(const T* X, const T* gx, long long q, long long qn) {
    const double d = (double)X[qn] - (double)X[q];
    const double sg = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0);
    return sg * ((double)gx[q] - (double)gx[qn]);
}

// per-edge gradients in the weight maps' layout (gWf / gWs: the F- / S-axis maps, either may be nullptr)
template <typename T>
__global__ void k_gw(G2 g, const uint32_t* __restrict__ BF, const uint32_t* __restrict__ BS, const T* __restrict__ X, const T* __restrict__ gx,
                     T* __restrict__ gWf, T* __restrict__ gWs) {
    GRID_STRIDE(q, g.n) {
        const long long b = q / g.img, e = q - b * g.img;
        const int f = (int)(e % g.F), s = (int)(e / g.F);
        if (gWf && f < g.F - 1) gWf[q - (b * g.S + s)] = tape_bit(BF, q) ? T(0) : (T)edge_gw(X, gx, q, q + 1);
        if (gWs && s < g.S - 1) gWs[q - b * g.F] = tape_bit(BS, q) ? T(0) : (T)edge_gw(X, gx, q, q + g.F);
    }
}

__device__ __forceinline__ double block_sum(double v) {
    __shared__ double sm[32];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();                                                  // sm is reused by the block's next task
    if (l == 0) sm[w] = v;
    __syncthreads();
    v = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.0;
    if (w == 0) for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;                                                         // thread 0
}

// first stage of glam: task (b, axis, chunk) sums the (T-rounded) gw of the canonical elements [chunk GLAM_CHUNK, + GLAM_CHUNK) of
// image b along axis (0: the edge to (i + 1, j), 1: to (i, j + 1)); thread t takes elements t, t + 256, ... in order, then a fixed tree
template <typename T>
__global__ void k_glam_part(G2 g, int M, int N, int batch, long long nchunks, const uint32_t* __restrict__ BF, const uint32_t* __restrict__ BS,
                            const T* __restrict__ X, const T* __restrict__ gx, double* __restrict__ part) {
    const long long tasks = (long long)batch * 2 * nchunks;
    for (long long task = blockIdx.x; task < tasks; task += gridDim.x) {
        const long long k = task % nchunks, ba = task / nchunks;
        const int axis = (int)(ba & 1);
        const long long b = ba >> 1;
        const long long c1 = (k + 1) * GLAM_CHUNK < g.img ? (k + 1) * GLAM_CHUNK : g.img;
        double v = 0.0;
        for (long long c = k * GLAM_CHUNK + threadIdx.x; c < c1; c += blockDim.x) {
            const int i = (int)(c % M), j = (int)(c / M);
            if (axis == 0 ? i >= M - 1 : j >= N - 1) continue;
            const long long q = b * g.img + (g.row_major ? (long long)j + (long long)N * i : c);
            const bool along_f = (axis == 0) != (g.row_major != 0);      // axis 0 is F for column-major storage
            const long long qn = q + (along_f ? 1 : g.F);
            if (!tape_bit(along_f ? BF : BS, q)) v += (double)(T)edge_gw(X, gx, q, qn);
        }
        v = block_sum(v);
        if (threadIdx.x == 0) part[task] = v;
    }
}

__global__ void k_glam_final(int batch, long long nchunks, const double* __restrict__ part, double* __restrict__ glam) {
    for (int t = blockIdx.x; t < 2 * batch; t += gridDim.x) {
        double v = 0.0;
        for (long long k = threadIdx.x; k < nchunks; k += blockDim.x) v += part[(long long)t * nchunks + k];
        v = block_sum(v);
        if (threadIdx.x == 0) glam[t] = v;
    }
}

G2 geom(size_t M, size_t N, int batch, int row_major) {
    G2 g;
    g.F = (int)(row_major ? N : M); g.S = (int)(row_major ? M : N); g.M = (int)M; g.row_major = row_major ? 1 : 0;
    g.img = (long long)(M * N); g.n = g.img * batch;
    return g;
}

}  // namespace

size_t cp2_tape_bytes(size_t M, size_t N, int batch) {
    return 256 + 2 * ptvv::vjp_tape_set_bytes((long long)(M * N * (size_t)batch));
}

size_t ws_bytes_cp2_vjp(size_t M, size_t N, int batch) {
    const size_t n = M * N * (size_t)batch, nchunks = (M * N + GLAM_CHUNK - 1) / GLAM_CHUNK;
    return 3 * al256(n * sizeof(int)) + al256(3 * n * sizeof(long long)) + al256(2 * (size_t)batch * nchunks * sizeof(double));
}

template <typename T>
cudaError_t cp2_tape_tail(size_t M, size_t N, int batch, int row_major, const T* X, const T* const Uf[2], const T* const Us[2], const int* stopped,
                          int it_end, double lambda, bool weighted, const T* Wf, const T* Ws, void* tape, cudaStream_t st) {
    const G2 g = geom(M, N, batch, row_major);
    Cp2TapeHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = CP2_TAPE_MAGIC; h.elem = (int64_t)sizeof(T); h.M = (int64_t)M; h.N = (int64_t)N; h.batch = batch;
    h.row_major = g.row_major; h.weighted = weighted ? 1 : 0;
    cudaError_t e = cudaMemcpyAsync(tape, &h, sizeof(h), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    const size_t sb = ptvv::vjp_tape_set_bytes(g.n);
    uint32_t* BF = (uint32_t*)((char*)tape + 256);
    uint32_t* BS = (uint32_t*)((char*)tape + 256 + sb);
    const long long nwords = (g.n + 31) / 32;
    const unsigned grid = grid_for(nwords * 32);
    if (weighted) k_cp2_tape<T, true><<<grid, 256, 0, st>>>(g, X, Uf[0], Uf[1], Us[0], Us[1], stopped, it_end, T(0), Wf, Ws, BF, BS, nwords);
    else k_cp2_tape<T, false><<<grid, 256, 0, st>>>(g, X, Uf[0], Uf[1], Us[0], Us[1], stopped, it_end, (T)lambda, nullptr, nullptr, BF, BS, nwords);
    return cudaGetLastError();
}

const char* cp2_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, bool weighted, cudaStream_t st) {
    Cp2TapeHeader h;
    if (cudaMemcpyAsync(&h, tape, sizeof(h), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError(); return "cannot read the tape header";
    }
    if (h.magic != CP2_TAPE_MAGIC) return "not a CP2_TV tape";
    if (h.elem != (int64_t)elem) return "tape recorded with another dtype";
    if (h.M != (int64_t)M || h.N != (int64_t)N || h.batch != batch) return "tape recorded for another shape";
    if (h.row_major != (row_major ? 1 : 0)) return "tape recorded for another storage order";
    if (h.weighted != (weighted ? 1 : 0)) return weighted ? "tape recorded by the unweighted solver" : "tape recorded by the weighted solver";
    return nullptr;
}

template <typename T>
cudaError_t cp2_vjp_device(size_t M, size_t N, int batch, int row_major, const void* tape, const T* X, const T* gout, T* gY, T* gW1, T* gW2,
                           double* glam, void* ws, cudaStream_t st) {
    const G2 g = geom(M, N, batch, row_major);
    const size_t sb = ptvv::vjp_tape_set_bytes(g.n);
    const uint32_t* BF = (const uint32_t*)((const char*)tape + 256);
    const uint32_t* BS = (const uint32_t*)((const char*)tape + 256 + sb);
    const long long nchunks = (g.img + GLAM_CHUNK - 1) / GLAM_CHUNK;
    char* w = (char*)ws;
    int* P = (int*)w; w += al256((size_t)g.n * sizeof(int));
    int* cnt = (int*)w; w += al256((size_t)g.n * sizeof(int));
    int* emax = (int*)w; w += al256((size_t)g.n * sizeof(int));
    long long* acc = (long long*)w; w += al256(3 * (size_t)g.n * sizeof(long long));
    double* part = (double*)w;
    const unsigned grid = grid_for(g.n);
#define VTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
    VTRY(cudaMemsetAsync(cnt, 0, (size_t)g.n * sizeof(int), st));
    VTRY(cudaMemsetAsync(emax, 0x80, (size_t)g.n * sizeof(int), st));             // NO_EXP
    VTRY(cudaMemsetAsync(acc, 0, 3 * (size_t)g.n * sizeof(long long), st));
    k_cc_init<<<grid, 256, 0, st>>>(g, P);
    k_cc_union<<<grid, 256, 0, st>>>(g, BF, BS, P);
    k_cc_flatten<<<grid, 256, 0, st>>>(g, P);
    k_sum_scale<T><<<grid, 256, 0, st>>>(g, P, gout, cnt, emax);
    k_sum_add<T><<<grid, 256, 0, st>>>(g, P, gout, emax, acc);
    k_gx<T><<<grid, 256, 0, st>>>(g, P, cnt, emax, acc, gY);
    VTRY(cudaGetLastError());
    if (gW1 || gW2) {
        T* gWf = row_major ? gW2 : gW1;
        T* gWs = row_major ? gW1 : gW2;
        k_gw<T><<<grid, 256, 0, st>>>(g, BF, BS, X, gY, gWf, gWs);
        VTRY(cudaGetLastError());
    }
    if (glam) {
        const long long tasks = (long long)batch * 2 * nchunks;
        k_glam_part<T><<<(unsigned)(tasks < 132 * 16 ? tasks : 132 * 16), 256, 0, st>>>(g, (int)M, (int)N, batch, nchunks, BF, BS, X, gY, part);
        k_glam_final<<<(unsigned)(2 * batch < 132 * 16 ? 2 * batch : 132 * 16), 256, 0, st>>>(batch, nchunks, part, glam);
        VTRY(cudaGetLastError());
    }
#undef VTRY
    return cudaSuccess;
}

template cudaError_t cp2_tape_tail<double>(size_t, size_t, int, int, const double*, const double* const[2], const double* const[2], const int*,
                                           int, double, bool, const double*, const double*, void*, cudaStream_t);
template cudaError_t cp2_tape_tail<float>(size_t, size_t, int, int, const float*, const float* const[2], const float* const[2], const int*,
                                          int, double, bool, const float*, const float*, void*, cudaStream_t);
template cudaError_t cp2_vjp_device<double>(size_t, size_t, int, int, const void*, const double*, const double*, double*, double*, double*,
                                            double*, void*, cudaStream_t);
template cudaError_t cp2_vjp_device<float>(size_t, size_t, int, int, const void*, const float*, const float*, float*, float*, float*,
                                           double*, void*, cudaStream_t);

}  // namespace ptv
