// vjp.cu -- backward pass of the batched 1D TV-L1 prox over the fibers (nf, len, inc): gx = segment means of g, gw per edge
// (contract and work split: vjp_core.cuh).  A pure streaming computation; the forward kernels are not involved.
//
//   k_vjp_scan   pass 1, one lane per work item (a whole fiber, or one chunk of it), 32 items per warp scanning in lock step.  Strided
//                fibers (inc > 1): the items of a warp are adjacent fibers, so every row is one coalesced load, prefetched R rows ahead
//                into registers.  Contiguous fibers: the warp stages R rows x 32 items through a shared-memory tile (each item's rows are
//                64 contiguous bytes) and every lane reads its own column.
//   k_vjp_carry  pass 2 (chunked work only), one thread per chunk: the open segment that begins in it, its sum continued in order
//                through the following chunks.
//   k_vjp_fix    pass 3 (chunked work only), one thread per chunk: the open parts and the edges next to them.
// Chunks are used when there are too few fibers to fill the device (one long signal, a small batch); vjp_chunk_len() decides.
#include "ptv_internal.h"
#include "vjp_core.cuh"

namespace ptvv {

using ptv::KernelSpan;

constexpr int VJP_WARPS = 4;                                  // warps per block of the scan and fix-up kernels
template <typename T> constexpr int vjp_rows() { return 64 / (int)sizeof(T); }   // rows per tile / prefetch batch: 64 bytes per item

template <typename T> struct VjpArgs {
    const T* y; const T* g; T* gx; T* gw; const T* w; double lam;
    long long nf, inc; int len;
    const uint32_t* tf; const uint32_t* tu;    // tape-driven kernels (TAPE): the pass's segmentation tape instead of y and the weights
    __device__ long long base(long long f) const { return (f / inc) * inc * (long long)len + f % inc; }        // src/TVNDopt.cpp:184-188
    __device__ long long wbase(long long f) const { return (f / inc) * inc * (long long)(len - 1) + f % inc; }
    __device__ bool wpos(long long wb, int e) const { return w ? w[wb + (long long)e * inc] > T(0) : lam > 0.0; }
};

template <typename T> struct DevOut {
    T* px; T* pw; long long xb, wb, inc;
    __device__ void gx(int k, T v) { px[xb + (long long)k * inc] = v; }
    __device__ void gw(int e, T v) { if (pw) pw[wb + (long long)e * inc] = v; }
};

struct Item { long long f; int c, c0, c1; bool act; };
__device__ inline Item vjp_item(long long nf, int len, int C, int nc) {
    const long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // chunk-major: the lanes of a warp take adjacent fibers
    Item r;
    r.act = it < nf * nc;
    r.f = r.act ? it % nf : 0;
    r.c = r.act ? (int)(it / nf) : 0;
    r.c0 = r.c * C;
    r.c1 = min(len, r.c0 + C);
    return r;
}

// TAPE: "fused" and the sign of every edge come from the tape (vjp_core.cuh) instead of y and the weights; the tile and register
// slots of y[i + 1] and w[i] then carry the sign and the fused flag (as T: +1 / -1 / 0 and 1 / 0).  Same scan, same records.
template <typename T, bool TILE, bool TAPE>
__global__ void __launch_bounds__(32 * VJP_WARPS) k_vjp_scan(VjpArgs<T> a, int C, int nc, VjpRec* rec) {
    constexpr int R = TILE ? vjp_rows<T>() : 8;              // strided: every row is one coalesced load; 8 in flight per lane
    constexpr int TW = TILE ? VJP_WARPS : 1, TR = TILE ? R : 1;
    __shared__ T sg[TW][TR][33], sy[TW][TR][33], sw[TW][TR][33];        // [row][item], padded: conflict-free fills and reads
    const int lane = threadIdx.x & 31, wid = TILE ? threadIdx.x >> 5 : 0;
    const Item it = vjp_item(a.nf, a.len, C, nc);
    const long long xb = a.base(it.f), wb = a.wbase(it.f), inc = a.inc;
    const int len = a.len, n = it.act ? it.c1 - it.c0 : 0;
    DevOut<T> out{a.gx, a.gw, xb, wb, inc};
    VjpScan<T> sc;
    if (it.act) {
        if constexpr (TAPE) {
            sc.begin(it.c0, len, T(0), it.c0 > 0 && vjp_tape_fused(a.tf, a.tu, xb + (long long)(it.c0 - 1) * inc));
        } else {
            const T y0 = a.y[xb + (long long)it.c0 * inc];
            const bool ol = it.c0 > 0 && a.y[xb + (long long)(it.c0 - 1) * inc] == y0 && a.wpos(wb, it.c0 - 1);
            sc.begin(it.c0, len, y0, ol);
        }
    }
    const int nmax = (int)__reduce_max_sync(0xffffffffu, (unsigned)n);
    // The next batch of rows is requested before the current one is scanned, so its loads are in flight during the scan.
    if constexpr (TILE) {
        // inc == 1: tile column j = rows [r0, r0 + R) of lane j's item (g, w) and the same rows shifted by one (y[i + 1]); each lane
        // fetches R elements per array (CPI columns per request, 64 contiguous bytes each) into registers, then stores them to the tile
        constexpr int CPI = 32 / R;
        const int rr = lane % R, jj = lane / R;
        T pg[R], py[R], pw[R];
        auto fetch = [&](int r0) {
#pragma unroll
            for (int q = 0; q < R; q++) {
                const int j = q * CPI + jj;
                const long long sb = __shfl_sync(0xffffffffu, xb + it.c0, j);
                const long long swb = __shfl_sync(0xffffffffu, wb + it.c0, j);
                const int nj = __shfl_sync(0xffffffffu, n, j);
                const int rem = __shfl_sync(0xffffffffu, len - it.c0, j);       // rows of the fiber from the item's first row on
                const int k = r0 + rr;
                pg[q] = k < nj ? a.g[sb + k] : T(0);
                if constexpr (TAPE) {
                    const bool e = k < nj && k + 1 < rem;
                    py[q] = e ? (T)vjp_tape_sgn(a.tf, a.tu, sb + k) : T(0);
                    pw[q] = (e && vjp_tape_fused(a.tf, a.tu, sb + k)) ? T(1) : T(0);
                } else {
                    py[q] = (k < nj && k + 1 < rem) ? a.y[sb + k + 1] : T(0);
                    pw[q] = (a.w && k < nj && k + 1 < rem) ? a.w[swb + k] : T(0);
                }
            }
        };
        if (nmax > 0) fetch(0);
        for (int r0 = 0; r0 < nmax; r0 += R) {
            __syncwarp();
#pragma unroll
            for (int q = 0; q < R; q++) {
                const int j = q * CPI + jj;
                sg[wid][rr][j] = pg[q]; sy[wid][rr][j] = py[q]; sw[wid][rr][j] = pw[q];
            }
            __syncwarp();
            if (r0 + R < nmax) fetch(r0 + R);
            for (int k = 0; k < R; k++) {
                if (r0 + k < n) {
                    const int i = it.c0 + r0 + k;
                    const bool nl = i + 1 < len;
                    if constexpr (TAPE) {
                        const T sgn = sy[wid][k][lane];
                        sc.step(i, sg[wid][k][lane], nl && sw[wid][k][lane] > T(0), [&]() { return (double)sgn; }, out);
                    } else {
                        const bool wp = nl && (a.w ? sw[wid][k][lane] > T(0) : a.lam > 0.0);
                        sc.row(i, sg[wid][k][lane], sy[wid][k][lane], wp, out);
                    }
                }
            }
        }
    } else {
        // strided: the lanes' items are adjacent fibers, so each row is one coalesced request; two register batches alternate
        // (the weights are compared only when scanned: a comparison at fetch time would wait for the load)
        T ag[R], ay[R], aw[R], bg[R], by[R], bw[R];
        const T upos = a.lam > 0.0 ? T(1) : T(0);
        auto fetch = [&](int r0, T* rg, T* ry, T* rw) {
#pragma unroll
            for (int k = 0; k < R; k++) {
                const int i = it.c0 + r0 + k;
                const bool in = r0 + k < n, nl = in && i + 1 < len;
                rg[k] = in ? a.g[xb + (long long)i * inc] : T(0);
                if constexpr (TAPE) {
                    ry[k] = nl ? (T)vjp_tape_sgn(a.tf, a.tu, xb + (long long)i * inc) : T(0);
                    rw[k] = (nl && vjp_tape_fused(a.tf, a.tu, xb + (long long)i * inc)) ? T(1) : T(0);
                } else {
                    ry[k] = nl ? a.y[xb + (long long)(i + 1) * inc] : T(0);
                    rw[k] = nl ? (a.w ? a.w[wb + (long long)i * inc] : upos) : T(0);
                }
            }
        };
        auto scan = [&](int r0, const T* rg, const T* ry, const T* rw) {
#pragma unroll
            for (int k = 0; k < R; k++)
                if (r0 + k < n) {
                    if constexpr (TAPE) { const T sgn = ry[k]; sc.step(it.c0 + r0 + k, rg[k], rw[k] > T(0), [&]() { return (double)sgn; }, out); }
                    else sc.row(it.c0 + r0 + k, rg[k], ry[k], rw[k] > T(0), out);
                }
        };
        if (nmax > 0) fetch(0, ag, ay, aw);
        for (int r0 = 0; r0 < nmax; r0 += 2 * R) {
            if (r0 + R < nmax) fetch(r0 + R, bg, by, bw);
            scan(r0, ag, ay, aw);
            if (r0 + R < nmax) {
                if (r0 + 2 * R < nmax) fetch(r0 + 2 * R, ag, ay, aw);
                scan(r0 + R, bg, by, bw);
            }
        }
    }
    if (rec && it.act) sc.finish(rec[it.f * nc + it.c]);
}

template <typename T>
__global__ void __launch_bounds__(32 * VJP_WARPS) k_vjp_carry(VjpArgs<T> a, int C, int nc, const VjpRec* rec, VjpMeans* mm) {
    const Item it = vjp_item(a.nf, a.len, C, nc);
    if (!it.act) return;
    const long long xb = a.base(it.f), inc = a.inc;
    const T* g = a.g;
    VjpMeans* M = mm + it.f * nc;
    vjp_carry_from<T>(rec + it.f * nc, it.c, nc, C, a.len, [&](int i) { return g[xb + (long long)i * inc]; },
                      [&](int k) -> VjpMeans& { return M[k]; });
}

template <typename T, bool TAPE>
__global__ void __launch_bounds__(32 * VJP_WARPS) k_vjp_fix(VjpArgs<T> a, int C, int nc, const VjpRec* rec, const VjpMeans* mm) {
    const Item it = vjp_item(a.nf, a.len, C, nc);
    if (!it.act) return;
    const long long xb = a.base(it.f), wb = a.wbase(it.f), inc = a.inc, ri = it.f * nc + it.c;
    const VjpRec r = rec[ri];
    const double mnext = it.c + 1 < nc ? vjp_first_mean(rec[ri + 1], mm[ri + 1]) : 0.0;
    DevOut<T> out{a.gx, a.gw, xb, wb, inc};
    const T* y = a.y; const T* gx = a.gx;
    if constexpr (TAPE)
        vjp_fix_chunk_sg<T>(r, mm[ri], it.c0, it.c1, a.len, mnext, a.gw != nullptr,
                            [&](int e) { return vjp_tape_sgn(a.tf, a.tu, xb + (long long)e * inc); },
                            [&](int i) { return gx[xb + (long long)i * inc]; }, out);
    else
        vjp_fix_chunk<T>(r, mm[ri], it.c0, it.c1, a.len, mnext, a.gw != nullptr, [&](int i) { return y[xb + (long long)i * inc]; },
                         [&](int i) { return gx[xb + (long long)i * inc]; }, out);
}

static int g_vjp_clen = 0;                                     // tests: forced chunk length (0 = automatic)
void vjp_set_tuning(int clen) { g_vjp_clen = clen > 0 ? clen : 0; }

// Whole fibers when they alone fill the device (>= 32768 lanes) or are short; otherwise chunks of >= 256 rows, enough for about 65536
// work items.
int vjp_chunk_len(long long nf, int len) {
    if (g_vjp_clen > 0) return g_vjp_clen < len ? g_vjp_clen : len;
    if (nf >= 32768 || len <= 512) return len;
    const long long nc = (65536 + nf - 1) / nf;
    long long c = (len + nc - 1) / nc;
    if (c < 256) c = 256;
    return c < len ? (int)c : len;
}

size_t vjp_scratch_bytes(long long nf, int len) {
    if (nf <= 0 || len <= 0) return 0;
    const int C = vjp_chunk_len(nf, len);
    const long long nc = (len + C - 1) / C;
    return nc > 1 ? (size_t)(nf * nc) * (sizeof(VjpRec) + sizeof(VjpMeans)) : 0;
}

template <typename T, bool TAPE>
static cudaError_t vjp_launch(const VjpArgs<T>& a, void* scratch, cudaStream_t st) {
    const long long nf = a.nf, inc = a.inc;
    const int len = a.len;
    if (nf <= 0 || len <= 0) return cudaSuccess;
    const int C = vjp_chunk_len(nf, len);
    const int nc = (len + C - 1) / C;
    const long long items = nf * nc;
    const unsigned blocks = (unsigned)((items + 32 * VJP_WARPS - 1) / (32 * VJP_WARPS));
    VjpRec* rec = nc > 1 ? (VjpRec*)scratch : nullptr;
    VjpMeans* mm = nc > 1 ? (VjpMeans*)(rec + items) : nullptr;
    if (nc > 1 && !scratch) return cudaErrorInvalidValue;
    {
        KernelSpan span(inc == 1 ? ptv::KC_PROX_CONTIG : ptv::KC_PROX_STRIDED, 1, st);
        if (inc == 1) k_vjp_scan<T, true, TAPE><<<blocks, 32 * VJP_WARPS, 0, st>>>(a, C, nc, rec);
        else k_vjp_scan<T, false, TAPE><<<blocks, 32 * VJP_WARPS, 0, st>>>(a, C, nc, rec);
    }
    if (nc > 1) {
        KernelSpan span(ptv::KC_ELEMENTWISE, 2, st);
        k_vjp_carry<T><<<blocks, 32 * VJP_WARPS, 0, st>>>(a, C, nc, rec, mm);
        k_vjp_fix<T, TAPE><<<blocks, 32 * VJP_WARPS, 0, st>>>(a, C, nc, rec, mm);
    }
    return cudaGetLastError();
}

template <typename T>
cudaError_t vjp_fibers(const T* y, const T* g, T* gx, T* gw, long long nf, int len, long long inc, T lam, const T* lamv, void* scratch,
                       cudaStream_t st) {
    const VjpArgs<T> a{y, g, gx, gw, lamv, (double)lam, nf, inc, len, nullptr, nullptr};
    return vjp_launch<T, false>(a, scratch, st);
}

template <typename T>
cudaError_t vjp_fibers_tape(const uint32_t* F, const uint32_t* U, const T* g, T* gx, T* gw, long long nf, int len, long long inc,
                            void* scratch, cudaStream_t st) {
    const VjpArgs<T> a{nullptr, g, gx, gw, nullptr, 0.0, nf, inc, len, F, U};
    return vjp_launch<T, true>(a, scratch, st);
}

// The tape of y over the fibers (nf, len, inc) (nf a multiple of inc: the fibers cover the nf * len elements once): one warp per
// 32-element word, the words of the 256-byte padding written as 0.  LAMF: the penalty of fiber j is lamf[j / fpi] -- with fpi a
// multiple of inc a group of fibers is a range of epi = fpi len elements, so element i's is lamf[i / epi].
template <typename T, bool LAMF = false>
__global__ void k_fiber_tape(const T* __restrict__ y, long long n, int len, long long inc, double lam, const T* __restrict__ w,
                             uint32_t* __restrict__ F, uint32_t* __restrict__ U, long long nwords, const T* __restrict__ lamf, long long epi) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = w0; q < nwords; q += ws) {
        const long long i = q * 32 + lane;
        uint32_t f = 0, u = 0;
        if (i < n) vjp_tape_edge<T>(y, i, len, inc, LAMF ? (double)lamf[i / epi] : lam, w, f, u);
        const uint32_t bf = __ballot_sync(0xffffffffu, f), bu = __ballot_sync(0xffffffffu, u);
        if (lane == 0) { F[q] = bf; U[q] = bu; }
    }
}

template <typename T>
cudaError_t fiber_tape(const T* y, long long nf, int len, long long inc, T lam, const T* lamv, uint32_t* F, uint32_t* U, cudaStream_t st) {
    const long long n = nf * (long long)len;
    const long long nwords = (long long)(vjp_tape_set_bytes(n) / 4);
    if (nwords == 0) return cudaSuccess;
    long long blocks = (nwords * 32 + 255) / 256;
    if (blocks > 132LL * 16) blocks = 132LL * 16;
    KernelSpan span(ptv::KC_ELEMENTWISE, 1, st);
    k_fiber_tape<T><<<(unsigned)blocks, 256, 0, st>>>(y, n, len, inc, (double)lam, lamv, F, U, nwords, nullptr, 1);
    return cudaGetLastError();
}

template <typename T>
cudaError_t fiber_tape_lamf(const T* y, long long nf, int len, long long inc, const T* lamf, long long fpi, uint32_t* F, uint32_t* U,
                            cudaStream_t st) {
    const long long n = nf * (long long)len;
    const long long nwords = (long long)(vjp_tape_set_bytes(n) / 4);
    if (nwords == 0) return cudaSuccess;
    long long blocks = (nwords * 32 + 255) / 256;
    if (blocks > 132LL * 16) blocks = 132LL * 16;
    KernelSpan span(ptv::KC_ELEMENTWISE, 1, st);
    k_fiber_tape<T, true><<<(unsigned)blocks, 256, 0, st>>>(y, n, len, inc, 0.0, nullptr, F, U, nwords, lamf, fpi * (long long)len);
    return cudaGetLastError();
}

template cudaError_t vjp_fibers<double>(const double*, const double*, double*, double*, long long, int, long long, double, const double*,
                                        void*, cudaStream_t);
template cudaError_t vjp_fibers<float>(const float*, const float*, float*, float*, long long, int, long long, float, const float*, void*,
                                       cudaStream_t);
template cudaError_t vjp_fibers_tape<double>(const uint32_t*, const uint32_t*, const double*, double*, double*, long long, int, long long,
                                             void*, cudaStream_t);
template cudaError_t vjp_fibers_tape<float>(const uint32_t*, const uint32_t*, const float*, float*, float*, long long, int, long long,
                                            void*, cudaStream_t);
template cudaError_t fiber_tape<double>(const double*, long long, int, long long, double, const double*, uint32_t*, uint32_t*, cudaStream_t);
template cudaError_t fiber_tape<float>(const float*, long long, int, long long, float, const float*, uint32_t*, uint32_t*, cudaStream_t);
template cudaError_t fiber_tape_lamf<double>(const double*, long long, int, long long, const double*, long long, uint32_t*, uint32_t*, cudaStream_t);
template cudaError_t fiber_tape_lamf<float>(const float*, long long, int, long long, const float*, long long, uint32_t*, uint32_t*, cudaStream_t);

}  // namespace ptvv
