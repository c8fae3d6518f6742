// dr2_vjp.cu -- the exact backward passes of DR2_TV (DESIGN.md section 11), of the weighted DR2L1W_TV (section 12), of the N-D
// PDR_TV (section 13) and of the proximal Dykstra PD_TV / PD2_TV (section 14, at the end): a recorded forward that writes the
// segmentation tape of every prox pass, and the unrolled vector-Jacobian product driven by that tape.
//
// DR2_TV is a fixed, unconverged splitting (35 iterations and a final projection), so the gradient is the one of the function actually
// computed: the lane engine's schedule (solver.cu: dr2_lane_body), per image, storage type T, column prox P_c (axis 0, penalty w1) and
// row prox P_r (axis 1, w2):
//     t_0 = 2 mean(Y)                     k = 0: x1 = t_0 (the prox of a constant), k >= 1: x1 = P_c(t_k)
//     d = t_k - x1 ;  u = Y - (2 d - t_k) ;  x2 = P_r(u) ;  t_{k+1} = d + x2                       k = 0 .. K-1
//     final: x1 = P_c(t_K) ;  d = t_K - x1 ;  out = P_r(Y - d)
// Every prox has the Jacobian of vjp_core.cuh: the mean over each constant segment, S_p(g) for pass p.  For an upstream gradient G:
//     final:      a = S_R(G) ; gY = a ; g_t = S_C(a) - a
//     k = K-1..0: G = g_t ; a = S_R(G) ; gY = gY + a ; h = G - 2 a ; g_t = (a + h) - S_C(h)
//     start:      gY = (T)((double)gY + (2.0 * sum_image(g_t)) / (M N))
// (k = 0: S_C is the column mean when w1 > 0 and M > 1, else the identity -- the Jacobian of the prox at a constant image).  All
// combines in T with exactly these associations (-fmad=false); sum_image is a double sum in the fixed two-stage order below.
//
// Tape: a 256-byte header (Dr2TapeHeader), then 2K + 1 passes in execution order -- p = 0: row pass of k = 0; p = 2k - 1 / 2k: column /
// row pass of iteration k (k = K: the final pair) -- each two bitsets F, U (vjp_core.cuh) of vjp_tape_set_bytes(n) bytes.  The first
// column pass (a constant) is not recorded.
//
// Penalty gradients (glam, per image [cols, rows]): a pass's gw (vjp_core.cuh rule 4 for its upstream gradient) summed per image in
// double (two-stage: fixed blocks, then one block per image) and added to the image's accumulator in backward execution order; the
// column passes' upstream gradient is -h, so their sums enter negated; the k = 0 column pass contributes 0.  No atomics: a call's
// result does not depend on timing.
#include "ptv_internal.h"
#include "vjp_core.cuh"
#include <limits.h>
#include <stdint.h>
#include <string.h>
#include <vector>

namespace ptv {

static inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
static constexpr size_t DR2V_SCRATCH = (REDUCE_BLOCKS + 8) * sizeof(double);

struct Dr2TapeHeader {
    uint64_t magic;
    int64_t elem, M, N, batch, row_major, K, w1pos, w2pos;
    int64_t pad[23];
};
static_assert(sizeof(Dr2TapeHeader) == 256, "tape header is 256 bytes");
static constexpr uint64_t DR2_TAPE_MAGIC = 0x3150415432524432ull;          // "2DR2TAP1"

size_t dr2_tape_bytes(size_t M, size_t N, int batch, int maxit) {
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    return 256 + (size_t)(2 * K + 1) * 2 * ptvv::vjp_tape_set_bytes((long long)(M * N * (size_t)batch));
}
template <typename T> size_t ws_bytes_dr2_record(size_t M, size_t N, int batch) {
    return 8 * al256(M * N * (size_t)batch * sizeof(T)) + DR2V_SCRATCH;      // t, d, u, x + 4 arrays of staging for prox_fibers
}
template <typename T> size_t ws_bytes_dr2_vjp(size_t M, size_t N, int batch) {
    const long long n = (long long)(M * N * (size_t)batch);
    const size_t s1 = ptvv::vjp_scratch_bytes((long long)N * batch, (int)M), s2 = ptvv::vjp_scratch_bytes((long long)M * batch, (int)N);
    return 6 * al256((size_t)n * sizeof(T)) + al256(s1 > s2 ? s1 : s2) + DR2V_SCRATCH + al256((size_t)batch * sizeof(double));
}

static unsigned ew_grid(long long n) {
    long long b = (n + 1023) / 1024;
    if (b < 1) b = 1;
    if (b > 132LL * 32) b = 132LL * 32;
    return (unsigned)b;
}
#define GRID_STRIDE(q, n) for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < (n); q += (long long)gridDim.x * blockDim.x)

// ---------------------------------------------------------------- recorded forward: combines that write the tape of the pass they read
// One warp per 32-element tape word; lane j handles element 32 q + j.  The pass output x is read at i and at its successor i + inc.
// Column pass (FINAL = false): d = t - x1 ; u = Y - (2 d - t)     (FINAL): d = t - x1 ; u = Y - d        tape of x1, column geometry
template <typename T, bool FINAL>
__global__ void k_rec_cols(const T* __restrict__ x1, const T* __restrict__ t, const T* __restrict__ Y, T* __restrict__ d, T* __restrict__ u,
                           long long n, int len, long long inc, double lam, uint32_t* __restrict__ F, uint32_t* __restrict__ U, long long nwords) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = w0; q < nwords; q += ws) {
        const long long i = q * 32 + lane;
        uint32_t f = 0, uu = 0;
        if (i < n) {
            ptvv::vjp_tape_edge<T>(x1, i, len, inc, lam, (const T*)nullptr, f, uu);
            const T tv = t[i];
            const T dv = tv - x1[i];
            d[i] = dv;
            u[i] = FINAL ? Y[i] - dv : Y[i] - (T(2) * dv - tv);
        }
        const uint32_t bf = __ballot_sync(0xffffffffu, f), bu = __ballot_sync(0xffffffffu, uu);
        if (lane == 0) { F[q] = bf; U[q] = bu; }
    }
}
// Row pass: t' = d + x2 ; tape of x2, row geometry
template <typename T>
__global__ void k_rec_rows(const T* __restrict__ x2, const T* __restrict__ d, T* __restrict__ tn, long long n, int len, long long inc,
                           double lam, uint32_t* __restrict__ F, uint32_t* __restrict__ U, long long nwords) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = w0; q < nwords; q += ws) {
        const long long i = q * 32 + lane;
        uint32_t f = 0, uu = 0;
        if (i < n) {
            ptvv::vjp_tape_edge<T>(x2, i, len, inc, lam, (const T*)nullptr, f, uu);
            tn[i] = d[i] + x2[i];
        }
        const uint32_t bf = __ballot_sync(0xffffffffu, f), bu = __ballot_sync(0xffffffffu, uu);
        if (lane == 0) { F[q] = bf; U[q] = bu; }
    }
}

static void dr2_geoms(size_t M, size_t N, int batch, int row_major, FiberGeom& gc, FiberGeom& gr) {
    gc = row_major ? FiberGeom{(long long)N * batch, (int)M, (long long)N} : FiberGeom{(long long)N * batch, (int)M, 1};
    gr = row_major ? FiberGeom{(long long)M * batch, (int)N, 1} : FiberGeom{(long long)M * batch, (int)N, (long long)M};
}

template <typename T>
cudaError_t dr2_record_device(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit, void* tape, void* ws,
                              Engine eng, cudaStream_t st) {
    const long long n = (long long)(M * N * (size_t)batch);
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    const size_t ab = al256((size_t)n * sizeof(T)), sb = ptvv::vjp_tape_set_bytes(n);
    char* w = (char*)ws;
    T* t = (T*)w; w += ab;
    T* d = (T*)w; w += ab;
    T* u = (T*)w; w += ab;
    T* x = (T*)w; w += ab;
    T* scr = (T*)w; w += 4 * ab;
    double* scratch = (double*)w;
    FiberGeom gc, gr;
    dr2_geoms(M, N, batch, row_major, gc, gr);
    // the engine and the lane decision of dr2_device for the same arguments
    eng = lane_guard<T>(eng, Y, n, (double)(w1 > w2 ? w1 : w2), st);
    void* lscr = nullptr;
    const bool lane = dr2_lane_pick<T>(M, N, batch, row_major, Y, out, ws, w1, w2, eng, &lscr) != 0;
    auto prox = [&](const T* in, T* o, bool col) -> cudaError_t {
        const FiberGeom& g = col ? gc : gr;
        const T lam = col ? w1 : w2;
        if (lane) {
            KernelSpan sp(g.inc == 1 ? KC_PROX_CONTIG : KC_PROX_STRIDED, 1, st);
            return ptvl::lane_prox<T>(ptvl::LANE_PLAIN, in, nullptr, nullptr, o, g.nf, g.len, g.inc, lam, lscr, st);
        }
        return prox_fibers<T>(in, nullptr, IN_A, o, 0, g, lam, nullptr, eng, scr, st, 4 * n);
    };
    auto Fp = [&](int p) { return (uint32_t*)((char*)tape + 256 + (size_t)p * 2 * sb); };
    auto Up = [&](int p) { return (uint32_t*)((char*)tape + 256 + (size_t)p * 2 * sb + sb); };
    const long long nwords = (long long)(sb / 4);
    const unsigned gw = ew_grid(nwords * 32);
#define RTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
    Dr2TapeHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = DR2_TAPE_MAGIC; h.elem = (int64_t)sizeof(T); h.M = (int64_t)M; h.N = (int64_t)N; h.batch = batch; h.row_major = row_major ? 1 : 0;
    h.K = K; h.w1pos = w1 > T(0); h.w2pos = w2 > T(0);
    RTRY(cudaMemcpyAsync(tape, &h, sizeof(h), cudaMemcpyHostToDevice, st));
    RTRY(ew_image_means_x2<T>(Y, (long long)(M * N), batch, t, scratch, st));          // t = 2 mean
    RTRY(ew_dr_first<T>(Y, t, u, d, n, st));                                           // k = 0: d = t - t ; u = Y - (2 d - t)
    for (int k = 0; k <= K; k++) {
        const bool final = k == K;
        if (k > 0) {
            RTRY(prox(t, x, true));
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            if (final) k_rec_cols<T, true><<<gw, 256, 0, st>>>(x, t, Y, d, u, n, gc.len, gc.inc, (double)w1, Fp(2 * k - 1), Up(2 * k - 1), nwords);
            else k_rec_cols<T, false><<<gw, 256, 0, st>>>(x, t, Y, d, u, n, gc.len, gc.inc, (double)w1, Fp(2 * k - 1), Up(2 * k - 1), nwords);
            RTRY(cudaGetLastError());
        }
        if (final) {
            RTRY(prox(u, out, false));
            RTRY(ptvv::fiber_tape<T>(out, gr.nf, gr.len, gr.inc, w2, nullptr, Fp(2 * k), Up(2 * k), st));
        } else {
            RTRY(prox(u, x, false));
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            k_rec_rows<T><<<gw, 256, 0, st>>>(x, d, t, n, gr.len, gr.inc, (double)w2, Fp(2 * k), Up(2 * k), nwords);
            RTRY(cudaGetLastError());
        }
    }
    return cudaSuccess;
}

static const char* tape_check(uint64_t magic, const char* not_ours, const void* tape, size_t elem, size_t M, size_t N, int batch,
                              int row_major, int maxit, cudaStream_t st) {
    Dr2TapeHeader h;
    if (cudaMemcpyAsync(&h, tape, sizeof(h), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError(); return "cannot read the tape header";
    }
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    if (h.magic != magic) return not_ours;
    if (h.elem != (int64_t)elem) return "tape recorded with another dtype";
    if (h.M != (int64_t)M || h.N != (int64_t)N || h.batch != batch) return "tape recorded for another shape";
    if (h.row_major != (row_major ? 1 : 0)) return "tape recorded for another storage order";
    if (h.K != K) return "tape recorded with another iteration count";
    return nullptr;
}
const char* dr2_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, int maxit, cudaStream_t st) {
    return tape_check(DR2_TAPE_MAGIC, "not a DR2_TV tape", tape, elem, M, N, batch, row_major, maxit, st);
}

// ---------------------------------------------------------------- backward
__device__ __forceinline__ double dr2v_block_sum(double v) {
    __shared__ double sm[32];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) sm[w] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? sm[threadIdx.x] : 0.0;
    if (w == 0) for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    return v;   // valid in thread 0
}
// per-image sums, stage 1: block x of image y sums a grid-stride slice of the image into partial[y][x]
template <typename T>
__global__ void k_img_partial(const T* __restrict__ a, long long per, double* __restrict__ partial) {
    const T* img = a + (long long)blockIdx.y * per;
    double acc = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < per; q += (long long)gridDim.x * blockDim.x) acc += (double)img[q];
    acc = dr2v_block_sum(acc);
    if (threadIdx.x == 0) partial[(long long)blockIdx.y * gridDim.x + blockIdx.x] = acc;
}
// stage 2: one block per image sums its nblk partials; glam != nullptr: glam[2 b + axis] += sign * sum, else sums[b] = sum
__global__ void k_img_final(const double* __restrict__ partial, int nblk, int b0, double* __restrict__ sums, double* __restrict__ glam, int axis,
                            double sign) {
    double acc = 0.0;
    for (int q = threadIdx.x; q < nblk; q += blockDim.x) acc += partial[(long long)blockIdx.x * nblk + q];
    acc = dr2v_block_sum(acc);
    if (threadIdx.x == 0) {
        const int b = b0 + blockIdx.x;
        if (glam) glam[2 * b + axis] = glam[2 * b + axis] + sign * acc;
        else sums[b] = acc;
    }
}
template <typename T>
static cudaError_t img_sums(const T* a, long long per, int batch, double* scratch, double* sums, double* glam, int axis, double sign,
                            cudaStream_t st) {
    if (per <= 0) return cudaSuccess;
    int nblk = (int)((per + 2047) / 2048);
    if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    const int share = REDUCE_BLOCKS / (batch < REDUCE_BLOCKS ? batch : REDUCE_BLOCKS);
    if (nblk > share) nblk = share < 1 ? 1 : share;
    int per_launch = REDUCE_BLOCKS / nblk; if (per_launch < 1) per_launch = 1;
    KernelSpan span(KC_ELEMENTWISE, 2 * ((batch + per_launch - 1) / per_launch), st);
    for (int b0 = 0; b0 < batch; b0 += per_launch) {
        const int nb = batch - b0 < per_launch ? batch - b0 : per_launch;
        k_img_partial<T><<<dim3(nblk, nb), 256, 0, st>>>(a + (long long)b0 * per, per, scratch);
        k_img_final<<<nb, 256, 0, st>>>(scratch, nblk, b0, sums, glam, axis, sign);
    }
    return cudaGetLastError();
}

template <typename T> __global__ void k_b_final(const T* __restrict__ a, const T* __restrict__ sc, T* __restrict__ gY, T* __restrict__ g, long long n) {
    GRID_STRIDE(q, n) { const T av = a[q]; gY[q] = av; g[q] = sc[q] - av; }
}
template <typename T> __global__ void k_b_mid1(const T* __restrict__ G, const T* __restrict__ a, T* __restrict__ gY, T* __restrict__ h, long long n) {
    GRID_STRIDE(q, n) { const T av = a[q]; gY[q] = gY[q] + av; h[q] = G[q] - T(2) * av; }
}
template <typename T> __global__ void k_b_mid2(const T* __restrict__ a, const T* __restrict__ h, const T* __restrict__ sc, T* __restrict__ g, long long n) {
    GRID_STRIDE(q, n) g[q] = (a[q] + h[q]) - sc[q];
}
template <typename T> __global__ void k_b_start(T* __restrict__ gY, const double* __restrict__ sums, long long per, long long n) {
    GRID_STRIDE(q, n) gY[q] = (T)((double)gY[q] + (2.0 * sums[q / per]) / (double)per);
}

template <typename T>
cudaError_t dr2_vjp_device(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY, double* glam,
                           void* ws, cudaStream_t st) {
    const long long n = (long long)(M * N * (size_t)batch), per = (long long)(M * N);
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    const size_t ab = al256((size_t)n * sizeof(T)), sb = ptvv::vjp_tape_set_bytes(n);
    const size_t s1 = ptvv::vjp_scratch_bytes((long long)N * batch, (int)M), s2 = ptvv::vjp_scratch_bytes((long long)M * batch, (int)N);
    char* w = (char*)ws;
    T* g = (T*)w; w += ab;
    T* a = (T*)w; w += ab;
    T* h = (T*)w; w += ab;
    T* sc = (T*)w; w += ab;
    T* gwb = (T*)w; w += ab;
    T* zero = (T*)w; w += ab;
    void* vscr = w; w += al256(s1 > s2 ? s1 : s2);
    double* scratch = (double*)w; w += DR2V_SCRATCH;
    double* sums = (double*)w;
    FiberGeom gc, gr;
    dr2_geoms(M, N, batch, row_major, gc, gr);
    Dr2TapeHeader hd;                                  // read by the caller's check; the flags are needed here too
    RTRY(cudaMemcpyAsync(&hd, tape, sizeof(hd), cudaMemcpyDeviceToHost, st));
    RTRY(cudaStreamSynchronize(st));
    const long long ec = gc.nf / batch * (gc.len - 1), er = gr.nf / batch * (gr.len - 1);     // edges per image of either pass
    const char* tb = (const char*)tape + 256;
    auto Fp = [&](int p) { return (const uint32_t*)(tb + (size_t)p * 2 * sb); };
    auto Up = [&](int p) { return (const uint32_t*)(tb + (size_t)p * 2 * sb + sb); };
    T* gw = glam ? gwb : nullptr;
    const unsigned ge = ew_grid(n);
    auto vjp = [&](int p, const T* gin, T* gx, bool col, double sign) -> cudaError_t {
        const FiberGeom& G = col ? gc : gr;
        RTRY(ptvv::vjp_fibers_tape<T>(Fp(p), Up(p), gin, gx, gw, G.nf, G.len, G.inc, vscr, st));
        if (glam) RTRY(img_sums<T>(gw, col ? ec : er, batch, scratch, nullptr, glam, col ? 0 : 1, sign, st));
        return cudaSuccess;
    };
    if (glam) RTRY(cudaMemsetAsync(glam, 0, 2 * (size_t)batch * sizeof(double), st));
    // final pair: out = P_r(Y - d), d = t_K - P_c(t_K)
    RTRY(vjp(2 * K, gout, a, false, 1.0));
    RTRY(vjp(2 * K - 1, a, sc, true, 1.0));                 // upstream of the final column prox: +a
    { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_final<T><<<ge, 256, 0, st>>>(a, sc, gY, g, n); RTRY(cudaGetLastError()); }
    for (int k = K - 1; k >= 0; k--) {
        RTRY(vjp(2 * k, g, a, false, 1.0));
        { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_mid1<T><<<ge, 256, 0, st>>>(g, a, gY, h, n); RTRY(cudaGetLastError()); }
        if (k > 0) RTRY(vjp(2 * k - 1, h, sc, true, -1.0));  // upstream of the column prox: -h
        else {
            // the prox of the constant start image: every column one segment (w1 > 0), or the identity (w1 == 0); M == 1 is one sample
            RTRY(cudaMemsetAsync(zero, 0, (size_t)n * sizeof(T), st));
            RTRY(ptvv::vjp_fibers<T>(zero, h, sc, nullptr, gc.nf, gc.len, gc.inc, hd.w1pos ? T(1) : T(0), nullptr, vscr, st));
        }
        { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_mid2<T><<<ge, 256, 0, st>>>(a, h, sc, g, n); RTRY(cudaGetLastError()); }
    }
    RTRY(img_sums<T>(g, per, batch, scratch, sums, nullptr, 0, 0.0, st));
    { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_start<T><<<ge, 256, 0, st>>>(gY, sums, per, n); RTRY(cudaGetLastError()); }
    return cudaSuccess;
}

// ================================================================ DR2L1W_TV (DESIGN.md section 12)
// drw_device's iteration (solver.cu) on `batch` M x N images in either storage order, column prox P_c (fibers of length M, weights W1
// (M-1) x N per image), row prox P_r (length N, weights W2 M x (N-1)), per image, in its own association (chunk_core.cuh: apply_out,
// apply_out_any):
//     t = 2 mean(Y)
//     k = 0..K-1: x1 = P_c(t) ; s = 2 (t - x1) - t ; u = Y - s ; x2 = P_r(u) ; tw = (u - x2) - Y ; t = 0.5 (t + (-2 tw - s))
//     final:      x1 = P_c(t) ; s = t - x1 ; u = Y - s ; x2 = P_r(u) ; tw = (u - x2) - Y ; out = -s - tw
// In real arithmetic t' = t - x1 + x2 and out = x2: section 11's recurrence, so the backward is dr2_vjp_device's with every pass
// recorded.  Tape: the 256-byte header (own magic) and 2K + 2 passes -- p = 2k / 2k + 1: column / row pass of iteration k (k = K: the
// final pair) -- the column pass of k = 0 included (the prox of a constant image, whose Jacobian depends on which weights are zero) --
// each a pair of bitsets over all batch M N elements in storage order.  Row tapes are taken from x2 itself: out is x2 only in real
// arithmetic.  The start value term sums g per image (img_sums); the weight gradients need no sum across images.
// Weight gradients: per edge, acc = 0.0 ; acc = acc + sign * (double)gw_p over the passes in backward order (p = 2K + 1 .. 0), gW = (T)acc,
// gw_p the pass's VJP edge gradient (laid out like W1 / W2) for its upstream gradient: G and a for the final pair, g for the row passes
// and -h for the column passes of the loop (computed for +h, so sign -1).
static constexpr uint64_t DRW_TAPE_MAGIC = 0x31504154574c5244ull;          // "DRLWTAP1"

size_t drw_tape_bytes(size_t M, size_t N, int batch, int maxit) {
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    return 256 + (size_t)(2 * K + 2) * 2 * ptvv::vjp_tape_set_bytes((long long)(M * N * (size_t)batch));
}
template <typename T> size_t ws_bytes_drw_record(size_t M, size_t N, int batch) {
    return 8 * al256(M * N * (size_t)batch * sizeof(T)) + DR2V_SCRATCH;   // t, s, u, x + DrwPasses' staging: t1, t2, gathered weights, sparse results
}
template <typename T> size_t ws_bytes_drw_vjp(size_t M, size_t N, int batch) {
    const long long n = (long long)(M * N * (size_t)batch);
    const size_t s1 = ptvv::vjp_scratch_bytes((long long)N * batch, (int)M), s2 = ptvv::vjp_scratch_bytes((long long)M * batch, (int)N);
    return 5 * al256((size_t)n * sizeof(T)) + 2 * al256((size_t)n * sizeof(double)) + al256(s1 > s2 ? s1 : s2) + DR2V_SCRATCH +
           al256((size_t)batch * sizeof(double));
}

// Column pass: s = 2 (t - x1) - t (FINAL: s = t - x1) ; u = Y - s ; tape of x1 over the columns (length len, stride inc) with W1
template <typename T, bool FINAL>
__global__ void k_recw_cols(const T* __restrict__ x1, const T* __restrict__ t, const T* __restrict__ Y, const T* __restrict__ W1,
                            T* __restrict__ s, T* __restrict__ u, long long n, int len, long long inc, uint32_t* __restrict__ F,
                            uint32_t* __restrict__ U, long long nwords) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = w0; q < nwords; q += ws) {
        const long long i = q * 32 + lane;
        uint32_t f = 0, uu = 0;
        if (i < n) {
            ptvv::vjp_tape_edge<T>(x1, i, len, inc, 0.0, W1, f, uu);
            const T tv = t[i];
            const T d = tv - x1[i];
            const T sv = FINAL ? d : T(2) * d - tv;
            s[i] = sv;
            u[i] = Y[i] - sv;
        }
        const uint32_t bf = __ballot_sync(0xffffffffu, f), bu = __ballot_sync(0xffffffffu, uu);
        if (lane == 0) { F[q] = bf; U[q] = bu; }
    }
}
// Row pass: tw = (u - x2) - Y ; dst = 0.5 (t + (-2 tw - s)) (FINAL: dst = -s - tw) ; tape of x2 over the rows (stride inc, length len)
// with W2.  dst may be t.
template <typename T, bool FINAL>
__global__ void k_recw_rows(const T* __restrict__ x2, const T* __restrict__ u, const T* __restrict__ Y, const T* __restrict__ s, const T* t,
                            T* dst, const T* __restrict__ W2, long long n, int len, long long inc, uint32_t* __restrict__ F,
                            uint32_t* __restrict__ U, long long nwords) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = w0; q < nwords; q += ws) {
        const long long i = q * 32 + lane;
        uint32_t f = 0, uu = 0;
        if (i < n) {
            ptvv::vjp_tape_edge<T>(x2, i, len, inc, 0.0, W2, f, uu);
            const T sv = s[i];
            T tw = (u[i] - x2[i]) - Y[i];
            if (FINAL) dst[i] = -sv - tw;
            else { tw = T(-2) * tw - sv; dst[i] = T(0.5) * (t[i] + tw); }
        }
        const uint32_t bf = __ballot_sync(0xffffffffu, f), bu = __ballot_sync(0xffffffffu, uu);
        if (lane == 0) { F[q] = bf; U[q] = bu; }
    }
}

template <typename T>
cudaError_t drw_record_device(size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit, void* tape,
                              void* ws, Engine eng, cudaStream_t st) {
    const long long n = (long long)(M * N * (size_t)batch);
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    const size_t ab = al256((size_t)n * sizeof(T)), sb = ptvv::vjp_tape_set_bytes(n);
    char* w = (char*)ws;
    T* t = (T*)w; w += ab;
    T* s = (T*)w; w += ab;
    T* u = (T*)w; w += ab;
    T* x = (T*)w; w += ab;
    DrwPasses<T> P;                                  // the pass routes of drw_device; the gathered weights are written first, below
    void* stage = w; w += 4 * ab;
    double* scratch = (double*)w;
    auto Fp = [&](int p) { return (uint32_t*)((char*)tape + 256 + (size_t)p * 2 * sb); };
    auto Up = [&](int p) { return (uint32_t*)((char*)tape + 256 + (size_t)p * 2 * sb + sb); };
    const long long nwords = (long long)(sb / 4);
    const unsigned gw = ew_grid(nwords * 32);
#define RTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
    Dr2TapeHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = DRW_TAPE_MAGIC; h.elem = (int64_t)sizeof(T); h.M = (int64_t)M; h.N = (int64_t)N; h.batch = batch; h.row_major = row_major ? 1 : 0;
    h.K = K;
    RTRY(cudaMemcpyAsync(tape, &h, sizeof(h), cudaMemcpyHostToDevice, st));
    RTRY(P.init(M, N, batch, row_major, W1, W2, eng, stage, st));
    const FiberGeom gc = P.g[0], gr = P.g[1];
    RTRY(ew_image_means_x2<T>(Y, (long long)(M * N), batch, t, scratch, st));
    for (int k = 0; k <= K; k++) {
        const bool final = k == K;
        RTRY(P.run(0, t, nullptr, nullptr, IN_A, x, 0 /*OUT_X*/, st));
        { KernelSpan sp(KC_ELEMENTWISE, 1, st);
          if (final) k_recw_cols<T, true><<<gw, 256, 0, st>>>(x, t, Y, P.W[0], s, u, n, gc.len, gc.inc, Fp(2 * k), Up(2 * k), nwords);
          else k_recw_cols<T, false><<<gw, 256, 0, st>>>(x, t, Y, P.W[0], s, u, n, gc.len, gc.inc, Fp(2 * k), Up(2 * k), nwords);
          RTRY(cudaGetLastError()); }
        RTRY(P.run(1, u, nullptr, nullptr, IN_A, x, 0 /*OUT_X*/, st));
        { KernelSpan sp(KC_ELEMENTWISE, 1, st);
          if (final) k_recw_rows<T, true><<<gw, 256, 0, st>>>(x, u, Y, s, t, out, P.W[1], n, gr.len, gr.inc, Fp(2 * k + 1), Up(2 * k + 1), nwords);
          else k_recw_rows<T, false><<<gw, 256, 0, st>>>(x, u, Y, s, t, t, P.W[1], n, gr.len, gr.inc, Fp(2 * k + 1), Up(2 * k + 1), nwords);
          RTRY(cudaGetLastError()); }
    }
    return cudaSuccess;
}

const char* drw_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, int maxit, cudaStream_t st) {
    return tape_check(DRW_TAPE_MAGIC, "not a DR2L1W_TV tape", tape, elem, M, N, batch, row_major, maxit, st);
}

template <typename T> __global__ void k_acc(double* __restrict__ acc, const T* __restrict__ gw, long long n, double sign) {
    GRID_STRIDE(q, n) acc[q] = acc[q] + sign * (double)gw[q];
}
template <typename T> __global__ void k_round(const double* __restrict__ acc, T* __restrict__ gW, long long n) {
    GRID_STRIDE(q, n) gW[q] = (T)acc[q];
}

template <typename T>
cudaError_t drw_vjp_device(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY, T* gW1, T* gW2,
                           void* ws, cudaStream_t st) {
    const long long per = (long long)(M * N), n = per * batch;
    const long long e1 = (long long)(M - 1) * (long long)N * batch, e2 = (long long)M * (long long)(N - 1) * batch;   // edges of W1 / W2
    const int K = maxit <= 0 ? MAX_ITERS_DR : maxit;
    const size_t ab = al256((size_t)n * sizeof(T)), db = al256((size_t)n * sizeof(double)), sb = ptvv::vjp_tape_set_bytes(n);
    const size_t s1 = ptvv::vjp_scratch_bytes((long long)N * batch, (int)M), s2 = ptvv::vjp_scratch_bytes((long long)M * batch, (int)N);
    char* w = (char*)ws;
    T* g = (T*)w; w += ab;
    T* a = (T*)w; w += ab;
    T* h = (T*)w; w += ab;
    T* sc = (T*)w; w += ab;
    T* gwb = (T*)w; w += ab;
    double* acc1 = (double*)w; w += db;
    double* acc2 = (double*)w; w += db;
    void* vscr = w; w += al256(s1 > s2 ? s1 : s2);
    double* scratch = (double*)w; w += DR2V_SCRATCH;
    double* sums = (double*)w;
    FiberGeom gc, gr;
    dr2_geoms(M, N, batch, row_major, gc, gr);
    const bool want1 = gW1 && e1 > 0, want2 = gW2 && e2 > 0;
    const char* tb = (const char*)tape + 256;
    auto Fp = [&](int p) { return (const uint32_t*)(tb + (size_t)p * 2 * sb); };
    auto Up = [&](int p) { return (const uint32_t*)(tb + (size_t)p * 2 * sb + sb); };
    // pass p = 2k (column) / 2k + 1 (row): gx = S_p(gin); with its map requested, acc += sign * gw_p
    auto vjp = [&](int p, const T* gin, T* gx, double sign) -> cudaError_t {
        const bool col = (p & 1) == 0;
        const FiberGeom& G = col ? gc : gr;
        const bool want = col ? want1 : want2;
        RTRY(ptvv::vjp_fibers_tape<T>(Fp(p), Up(p), gin, gx, want ? gwb : nullptr, G.nf, G.len, G.inc, vscr, st));
        if (want) {
            const long long ne = col ? e1 : e2;
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            k_acc<T><<<ew_grid(ne), 256, 0, st>>>(col ? acc1 : acc2, gwb, ne, sign);
            RTRY(cudaGetLastError());
        }
        return cudaSuccess;
    };
    if (want1) RTRY(cudaMemsetAsync(acc1, 0, (size_t)e1 * sizeof(double), st));
    if (want2) RTRY(cudaMemsetAsync(acc2, 0, (size_t)e2 * sizeof(double), st));
    const unsigned ge = ew_grid(n);
    RTRY(vjp(2 * K + 1, gout, a, 1.0));                     // final pair: out = P_r(u), u = Y - t + P_c(t)
    RTRY(vjp(2 * K, a, sc, 1.0));                          // upstream of the final column prox: +a
    { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_final<T><<<ge, 256, 0, st>>>(a, sc, gY, g, n); RTRY(cudaGetLastError()); }
    for (int k = K - 1; k >= 0; k--) {
        RTRY(vjp(2 * k + 1, g, a, 1.0));
        { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_mid1<T><<<ge, 256, 0, st>>>(g, a, gY, h, n); RTRY(cudaGetLastError()); }
        RTRY(vjp(2 * k, h, sc, -1.0));                     // upstream of the column prox: -h
        { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_mid2<T><<<ge, 256, 0, st>>>(a, h, sc, g, n); RTRY(cudaGetLastError()); }
    }
    RTRY(img_sums<T>(g, per, batch, scratch, sums, nullptr, 0, 0.0, st));
    { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_b_start<T><<<ge, 256, 0, st>>>(gY, sums, per, n); RTRY(cudaGetLastError()); }
    if (want1) { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_round<T><<<ew_grid(e1), 256, 0, st>>>(acc1, gW1, e1); RTRY(cudaGetLastError()); }
    if (want2) { KernelSpan sp(KC_ELEMENTWISE, 1, st); k_round<T><<<ew_grid(e2), 256, 0, st>>>(acc2, gW2, e2); RTRY(cudaGetLastError()); }
    return cudaSuccess;
#undef RTRY
}

// ================================================================ PDR_TV (DESIGN.md section 13)
// pdr_device (solver.cu) with k = npen terms, kk = (T)k, P_i the 1D prox along axis dims[i] with the scaled penalty lam_i, in T:
//     z_i = Y ;  j = 0..K-1:  p_i = P_i(z_i) ; q = sum_i p_i / kk ; x = sum_i z_i / kk ; z_i = z_i + ((2 q - x) - p_i)     out = x (j = K-1)
// The last iteration's passes do not reach out, so only the (K - 1) npen passes of j = 0..K-2 are recorded (pass p = j npen + i, after
// the 256-byte header).  Backward for the upstream gradient G, in T with exactly these associations (sums term by term, i in order):
//     v = G / kk ; gz_i = v                                                               (k_pdrv, start)
//     j = K-2..0:  s = (gz_0 + gz_1) + ... ; sk = s / kk ; h = 2 sk - gz_0
//                  i = 0..k-1:  gz_i = (gz_i - sk) + S_{j,i}(h) ; h = 2 sk - gz_{i+1}   (one VJP pass, then k_pdrv; the last term's step
//                                                                                         forms the next iteration's s, sk and h)
//     gY = (gz_0 + gz_1) + ...
// Penalty gradients: glam_i = 0.0 ; glam_i = glam_i + sum(gw_{j,i}) for j = K-2..0, gw_{j,i} the edge gradients (vjp_core.cuh rule 4) of
// pass (j, i) for its upstream gradient h, each sum img_sums' fixed two-stage double sum.  No atomics.
struct PdrTapeHeader {
    uint64_t magic;
    int32_t elem, K, npen, nds;
    int32_t ns[PDR_TAPE_MAX_DIMS];
    uint8_t axis[64];                                                       // 0-based axis of each term
    int32_t cap;                                                            // PD_TV / PD2_TV: the capacity in iterations; PDR_TV: 0
    int32_t batch;                                                          // the batched tapes (section 16): the items; else 0
    uint8_t pad[256 - 8 - 16 - 4 * PDR_TAPE_MAX_DIMS - 64 - 4 - 4];
};
static_assert(sizeof(PdrTapeHeader) == 256, "tape header is 256 bytes");

// What tells the three N-D tapes apart, by NdSolver: the magic, the refusal of another solver's tape, the default maxIters
struct NdTapeKind { uint64_t magic; const char* not_ours; int default_iters; };
static const NdTapeKind ND_TAPE[3] = {
    {0x3150415454324450ull, "not a PD2_TV tape", MAX_ITERS_PD},             // "PD2TTAP1"
    {0x3150415456544450ull, "not a PD_TV tape", MAX_ITERS_PD},              // "PDTVTAP1"
    {0x3150415452524450ull, "not a PDR_TV tape", MAX_ITERS_DR},             // "PDRRTAP1"
};
// the capacity in iterations
// the batched PD2_TV / PD_TV tapes (section 16), by NdSolver
static const NdTapeKind ND_TAPE_B[2] = {
    {0x3150415442324450ull, "not a batched PD2_TV tape", MAX_ITERS_PD},     // "PD2BTAP1"
    {0x3150415442544450ull, "not a batched PD_TV tape", MAX_ITERS_PD},      // "PDTBTAP1"
};
static int nd_cap(NdSolver s, int maxIters) { return maxIters <= 0 ? ND_TAPE[s].default_iters : maxIters; }
// the iterations the recorded passes come from: PDR_TV runs its capacity, PD_TV and PD2_TV what their stop rule let run
static int nd_K(NdSolver s, int maxIters, int iters) { return s == ND_PDR ? nd_cap(s, maxIters) : iters; }
// the passes of K iterations that reach the output (sections 13 and 14)
static unsigned long long nd_passes(NdSolver s, int npen, int K) {
    const unsigned long long k = (unsigned long long)K;
    switch (s) {
    case ND_PD2: return npen == 1 ? (K > 0 ? 1 : 0) : 2 * k;
    case ND_PD: return k * (unsigned long long)npen;
    default: return (unsigned long long)(K - 1) * (unsigned long long)npen;
    }
}

size_t nd_tape_head_bytes(int batch) { return 256 + (batch > 0 ? al256((size_t)batch * sizeof(int32_t)) : 0); }

// head + passes x two bitsets of n-element passes (batch >= 1: n batch elements), in 64-bit arithmetic; 0 when that does not fit in size_t
size_t nd_tape_bytes(NdSolver s, const int* ns, int nds, int npen, int maxIters, int batch) {
    NdTerms t;
    nd_terms(ns, nds, 0, nullptr, &t);
    if (batch > 0 && t.n > LLONG_MAX / batch) return 0;
    const unsigned long long passes = nd_passes(s, npen, nd_cap(s, maxIters));
    const unsigned long long set2 = 2ull * (unsigned long long)ptvv::vjp_tape_set_bytes(t.n * (batch > 0 ? batch : 1));
    const size_t head = nd_tape_head_bytes(batch);
    if (set2 && passes > (SIZE_MAX - head) / set2) return 0;
    return head + (size_t)(passes * set2);
}

template <typename T> cudaError_t nd_tape_pass(void* passes, long long cap_n, long long p, const T* y, FiberGeom g, T lam, cudaStream_t st,
                                               const T* lamf, long long fpi) {
    const size_t sb = ptvv::vjp_tape_set_bytes(cap_n);
    uint32_t* F = (uint32_t*)((char*)passes + (size_t)p * 2 * sb);
    if (lamf) return ptvv::fiber_tape_lamf<T>(y, g.nf, g.len, g.inc, lamf, fpi, F, F + sb / 4, st);
    return ptvv::fiber_tape<T>(y, g.nf, g.len, g.inc, lam, nullptr, F, F + sb / 4, st);
}
template <typename T> cudaError_t pdr_tape_pass(void* tape, long long n, long long p, const T* y, FiberGeom g, T lam, cudaStream_t st) {
    return nd_tape_pass<T>((char*)tape + 256, n, p, y, g, lam, st);
}

// K: the iterations recorded; cap: the capacity (PDR_TV, whose K is its capacity: 0)
static PdrTapeHeader nd_header(NdSolver s, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters) {
    PdrTapeHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = ND_TAPE[s].magic; h.elem = (int32_t)elem; h.K = nd_K(s, maxIters, iters); h.npen = npen; h.nds = nds;
    h.cap = s == ND_PDR ? 0 : nd_cap(s, maxIters);
    for (int i = 0; i < nds; i++) h.ns[i] = ns[i];
    for (int i = 0; i < npen; i++) h.axis[i] = (uint8_t)(int)(dims[i] - 1);
    return h;
}

cudaError_t nd_tape_header(NdSolver s, void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters,
                           cudaStream_t st) {
    const PdrTapeHeader h = nd_header(s, elem, ns, nds, npen, dims, maxIters, iters);
    return cudaMemcpyAsync(tape, &h, sizeof(h), cudaMemcpyHostToDevice, st);
}

// magic (not_ours when it is not this solver's), dtype, shape, terms, capacity, K
const char* nd_tape_check(NdSolver s, const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                          int iters, cudaStream_t st) {
    PdrTapeHeader h;
    if (cudaMemcpyAsync(&h, tape, sizeof(h), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError(); return "cannot read the tape header";
    }
    const PdrTapeHeader w = nd_header(s, elem, ns, nds, npen, dims, maxIters, iters);
    if (h.magic != w.magic) return ND_TAPE[s].not_ours;
    if (h.elem != w.elem) return "tape recorded with another dtype";
    if (h.nds != w.nds || memcmp(h.ns, w.ns, sizeof(h.ns)) != 0) return "tape recorded for another shape";
    if (h.npen != w.npen || memcmp(h.axis, w.axis, sizeof(h.axis)) != 0) return "tape recorded with other penalty terms";
    if (h.cap != w.cap) return "tape recorded with another maxIters";
    if (h.K != w.K) return "tape recorded with another iteration count";
    return nullptr;
}

// The batched tape (section 16): the header with the batched magic, K = the largest item K and `batch`, then the K table
static PdrTapeHeader nd_header_batched(NdSolver s, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, int batch,
                                       int Kmax) {
    PdrTapeHeader h = nd_header(s, elem, ns, nds, npen, dims, maxIters, Kmax);
    h.magic = ND_TAPE_B[s].magic;
    h.batch = batch;
    return h;
}

cudaError_t nd_tape_header_batched(NdSolver s, void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                                   int batch, const double* info, cudaStream_t st) {
    std::vector<char> head(nd_tape_head_bytes(batch), 0);
    int32_t* K = (int32_t*)(head.data() + 256);
    int Kmax = 0;
    for (int b = 0; b < batch; b++) { K[b] = (int32_t)info[3 * (size_t)b + INFO_ITERS]; if (K[b] > Kmax) Kmax = K[b]; }
    const PdrTapeHeader h = nd_header_batched(s, elem, ns, nds, npen, dims, maxIters, batch, Kmax);
    memcpy(head.data(), &h, sizeof(h));
    // pageable source: the copy is staged before the call returns
    return cudaMemcpyAsync(tape, head.data(), head.size(), cudaMemcpyHostToDevice, st);
}

// magic, dtype, shape, terms, capacity, batch, then the K table (every K in 1..cap, the largest the header's K), read back together
const char* nd_tape_check_batched(NdSolver s, const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims,
                                  int maxIters, int batch, int* K, cudaStream_t st) {
    std::vector<char> head(nd_tape_head_bytes(batch));
    if (cudaMemcpyAsync(head.data(), tape, head.size(), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError(); return "cannot read the tape header";
    }
    PdrTapeHeader h;
    memcpy(&h, head.data(), sizeof(h));
    const PdrTapeHeader w = nd_header_batched(s, elem, ns, nds, npen, dims, maxIters, batch, h.K);
    if (h.magic != w.magic) return ND_TAPE_B[s].not_ours;
    if (h.elem != w.elem) return "tape recorded with another dtype";
    if (h.nds != w.nds || memcmp(h.ns, w.ns, sizeof(h.ns)) != 0) return "tape recorded for another shape";
    if (h.npen != w.npen || memcmp(h.axis, w.axis, sizeof(h.axis)) != 0) return "tape recorded with other penalty terms";
    if (h.cap != w.cap) return "tape recorded with another maxIters";
    if (h.batch != w.batch) return "tape recorded for another batch";
    int Kmax = 0;
    memcpy(K, head.data() + 256, (size_t)batch * sizeof(int32_t));
    for (int b = 0; b < batch; b++) {
        if (K[b] < 1 || K[b] > h.cap) return "tape holds an invalid iteration count";
        if (K[b] > Kmax) Kmax = K[b];
    }
    if (Kmax != h.K) return "tape holds an invalid iteration count";
    return nullptr;
}

template <typename T> struct PdrvPtrs { T* gz[64]; };

// The backward workspace of the three solvers, in order: npen arrays a.gz (PD2_TV: gp, and gq when npen = 2), Sk (PD_TV: Gk; PD2_TV
// with npen = 1: gq), h, sc, gw (only when glam is wanted), the VJP scratch of the largest term, the double sums.  Returns its size
// and, unless ws is nullptr, splits ws into *L.
// batch = 0 (the single-item entry points): the double sums are REDUCE_BLOCKS + 8 doubles, and PD_TV / PD2_TV's one item keeps its slot
// table and slot map in the last 8.  batch >= 1 (section 16): every array holds the whole batch, the double sums one set of
// REDUCE_BLOCKS per item, then the device copies of the slot table and of the slot map.
template <typename T> struct NdVjpWs {
    PdrvPtrs<T> a;
    T *Sk, *h, *sc, *gw;
    void* vscr;
    double* scratch;
    int *dslots, *dmap;
};
template <typename T> static size_t nd_vjp_ws(const NdTerms& t, int npen, bool want_glam, char* ws, NdVjpWs<T>* L, int batch = 0) {
    const int nb = batch > 0 ? batch : 1;
    const size_t ab = al256((size_t)(t.n * nb) * sizeof(T));
    size_t vs = 0;
    for (int i = 0; i < npen; i++) {
        const size_t b = ptvv::vjp_scratch_bytes(t.g[i].nf * nb, t.g[i].len);
        if (b > vs) vs = b;
    }
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = ws ? ws + off : nullptr; off += bytes; return p; };
    for (int i = 0; i < npen; i++) L->a.gz[i] = (T*)take(ab);
    L->Sk = (T*)take(ab);
    L->h = (T*)take(ab);
    L->sc = (T*)take(ab);
    L->gw = want_glam ? (T*)take(ab) : nullptr;
    L->vscr = take(al256(vs));
    L->scratch = (double*)take(batch > 0 ? al256((size_t)batch * REDUCE_BLOCKS * sizeof(double)) : DR2V_SCRATCH);
    if (batch > 0) {
        L->dslots = (int*)take(al256((size_t)batch * sizeof(int)));
        L->dmap = (int*)take(al256((size_t)batch * sizeof(int)));
    } else {
        L->dslots = ws ? (int*)(L->scratch + REDUCE_BLOCKS) : nullptr;
        L->dmap = ws ? L->dslots + 1 : nullptr;
    }
    return off;
}
template <typename T> size_t ws_bytes_nd_vjp(const NdTerms& t, int npen, bool want_glam, int batch) {
    NdVjpWs<T> L;
    return nd_vjp_ws<T>(t, npen, want_glam, nullptr, &L, batch);
}

// start: v = G / kk, every gz_l = v.  Else the step after term i's VJP pass (result sc): gz_i = (gz_i - sk) + sc, then h = 2 sk - gz_{i+1}
// for the next term.  After the last term (and at the start): s = (gz_0 + gz_1) + ... ; more: sk = s / kk, h = 2 sk - gz_0 ; else gY = s.
template <typename T>
__global__ void k_pdrv(PdrvPtrs<T> a, int npen, int i, bool start, bool more, const T* __restrict__ G, const T* __restrict__ sc,
                       T* __restrict__ Sk, T* __restrict__ h, T* __restrict__ gY, long long n) {
    const T kk = (T)npen;
    GRID_STRIDE(q, n) {
        T v;
        if (start) {
            v = G[q] / kk;
            for (int l = 0; l < npen; l++) a.gz[l][q] = v;
        } else {
            const T sk = Sk[q];
            v = (a.gz[i][q] - sk) + sc[q];
            a.gz[i][q] = v;
            if (i + 1 < npen) { h[q] = T(2) * sk - a.gz[i + 1][q]; continue; }
        }
        // every gz_l holds its new value here; the last term's (all of them at the start) is v
        auto cur = [&](int l) { return (start || l == npen - 1) ? v : a.gz[l][q]; };
        T s = cur(0);
        for (int l = 1; l < npen; l++) s = s + cur(l);
        if (more) {
            const T sk = s / kk;
            Sk[q] = sk;
            h[q] = T(2) * sk - cur(0);
        } else {
            gY[q] = s;
        }
    }
}

// ================================================================ PD_TV and PD2_TV (DESIGN.md section 14)
// Both are the solvers of solver.cu themselves; the function differentiated is K iterations, K = the count the forward ran (info[0],
// the header's K): the stop test only picks K.  P_i is the 1D prox along axis dims[i], S_{j,i} its segment-mean Jacobian.
// PD_TV (pd_device, k = npen terms, kk = (T)k, lam_i scaled by k), all K npen passes reach out (pass p = j npen + i):
//     z_i = Y ;  j = 0..K-1:  p_i = P_i(z_i) ; x = ((0 + p_0 / kk) + p_1 / kk) + ... ; z_i = z_i + (x - p_i)       out = x (j = K-1)
//   backward, in T (sums term by term, i in order):
//     a_i = 0 ; gk = G / kk ; h = gk - 0                                                    (the start values, nd_vjp_items)
//     j = K-1..0:  i = 0..k-1:  a_i = a_i + S_{j,i}(h) ; h = gk - a_{i+1}     (one VJP pass, then k_pdv; after the last term:
//                  s = (a_0 + a_1) + ... ; j > 0: gk = s / kk, h = gk - a_0 ; j = 0: gY = s)
// PD2_TV (pd2_device, npen <= 2, penalties as given), passes 2j (z = P_0(x + p)) and 2j + 1 (x' = P_1(z + q)); npen = 1: one
// iteration, x' = z, pass 0.  Backward with the adjoints (gx, gp, gq) of (x', p', q') = (G, 0, 0); after the first step gx == gp, so
// one array gp holds both:
//     gp = 0 ; gq = 0 ; h = G - 0                                                           (the start values, nd_vjp_items)
//     j = K-1..0:  [npen = 2: gv = S_1(h) ; gq = gq + gv ; h = gq - gp                                      (k_pd2v, mode 1)]
//                  gu = S_0(h) ; gp = gp + gu ; j > 0: h = gp - gq ; j = 0: gY = gp                           (mode 2)
// Penalty gradients: glam_i = 0.0 ; glam_i = glam_i + sum(gw) per pass of term i in backward order, gw the pass's edge gradients for
// its upstream gradient h, each sum img_sums' fixed two-stage double sum.  No atomics.

// The step after term i's VJP pass (result sc): a_i = a_i + sc, then h = gk - a_{i+1} for the next term; after the last term
// s = (a_0 + a_1) + ... ; more: gk = s / kk, h = gk - a_0 ; else gY = s.
template <typename T>
__global__ void k_pdv(PdrvPtrs<T> a, int npen, int i, bool more, const T* __restrict__ sc, T* __restrict__ Gk, T* __restrict__ h,
                      T* __restrict__ gY, long long n) {
    const T kk = (T)npen;
    GRID_STRIDE(q, n) {
        const T v = a.gz[i][q] + sc[q];
        a.gz[i][q] = v;
        if (i + 1 < npen) { h[q] = Gk[q] - a.gz[i + 1][q]; continue; }
        T s = npen == 1 ? v : a.gz[0][q];
        for (int l = 1; l < npen; l++) s = s + (l == npen - 1 ? v : a.gz[l][q]);
        if (more) {
            const T gk = s / kk;
            Gk[q] = gk;
            h[q] = gk - (npen == 1 ? v : a.gz[0][q]);
        } else {
            gY[q] = s;
        }
    }
}

// mode 1 (after P_1's VJP, sc = gv): gq = gq + gv, h = gq - gp.  2 (after P_0's VJP, sc = gu): gp = gp + gu; more: h = gp - gq ; else
// gY = gp.
template <typename T>
__global__ void k_pd2v(int mode, bool more, const T* __restrict__ sc, T* __restrict__ gp, T* __restrict__ gq, T* __restrict__ h,
                       T* __restrict__ gY, long long n) {
    GRID_STRIDE(q, n) {
        if (mode == 1) {
            const T v = gq[q] + sc[q];
            gq[q] = v;
            h[q] = v - gp[q];
        } else {
            const T v = gp[q] + sc[q];
            if (more) { gp[q] = v; h[q] = v - gq[q]; }
            else gY[q] = v;
        }
    }
}

// glam[slots[s] npen + i] += the sum of slot s's partials (k_img_final's order and arithmetic, per item)
__global__ void k_item_final(const double* __restrict__ partial, int nblk, const int* __restrict__ slots, double* __restrict__ glam, int npen,
                             int i) {
    double acc = 0.0;
    for (int q = threadIdx.x; q < nblk; q += blockDim.x) acc += partial[(long long)blockIdx.x * nblk + q];
    acc = dr2v_block_sum(acc);
    if (threadIdx.x == 0) {
        double* g = glam + (long long)slots[blockIdx.x] * npen + i;
        *g = *g + 1.0 * acc;
    }
}
__global__ void k_scale(double* __restrict__ a, long long n, double f) { GRID_STRIDE(q, n) a[q] = a[q] * f; }

// PD_TV / PD2_TV, single-item (batch = 1) or batched (section 16): the recurrences above per item, item b over its own K_b = Kb[b].
// tb: the tape's first pass.  The adjoint arrays keep the forward's slot order (nd_slots); going down from the largest K, the items with
// K_b = j + 1 join at iteration j with the start values, the others moving to their new slots through sc.  Each pass's edge gradients
// are summed per item, into glam[b npen + i] (PD_TV: of the scaled penalties).
template <typename T>
static cudaError_t nd_vjp_items(NdSolver s, const NdTerms& t, int npen, int batch, const int* Kb, const char* tb, const T* gout, T* gY,
                                double* glam, const NdVjpWs<T>& L, cudaStream_t st) {
#define RTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
    const long long n = t.n;
    const size_t sb = ptvv::vjp_tape_set_bytes(n * batch);
    const T kk = (T)npen;
    int Kmax = 0;
    for (int b = 0; b < batch; b++) if (Kb[b] > Kmax) Kmax = Kb[b];
    // the carried state and how a joining item starts it
    T* arr[66]; int init[66]; int narr = 0;
    T* gp = L.a.gz[0];
    T* gq = npen >= 2 ? L.a.gz[1] : L.Sk;
    if (s == ND_PD) {
        for (int i = 0; i < npen; i++) { arr[narr] = L.a.gz[i]; init[narr++] = 0; }
        arr[narr] = L.Sk; init[narr++] = 1;
        arr[narr] = L.h; init[narr++] = 2;
    } else {
        arr[narr] = gp; init[narr++] = 0;
        arr[narr] = gq; init[narr++] = 0;
        arr[narr] = L.h; init[narr++] = 3;
    }
    std::vector<int> slots(batch), prev(batch), map(batch);
    int m = 0;
    long long nm = 0;
    auto pass = [&](long long p, int i) -> cudaError_t {
        const FiberGeom& g = t.g[i];
        const uint32_t* F = (const uint32_t*)(tb + (size_t)p * 2 * sb);
        RTRY(ptvv::vjp_fibers_tape<T>(F, F + sb / 4, L.h, L.sc, L.gw, g.nf * m, g.len, g.inc, L.vscr, st));
        const long long per = g.nf * (long long)(g.len - 1);
        if (glam && per > 0) {
            int nblk = (int)((per + 2047) / 2048);
            if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
            KernelSpan span(KC_ELEMENTWISE, 1 + (m + 65534) / 65535, st);
            for (int s0 = 0; s0 < m; s0 += 65535) {
                const int ny = m - s0 < 65535 ? m - s0 : 65535;
                k_img_partial<T><<<dim3(nblk, ny), 256, 0, st>>>(L.gw + (long long)s0 * per, per, L.scratch + (long long)s0 * nblk);
            }
            k_item_final<<<m, 256, 0, st>>>(L.scratch, nblk, L.dslots, glam, npen, i);
            RTRY(cudaGetLastError());
        }
        return cudaSuccess;
    };
    for (int j = Kmax - 1; j >= 0; j--) {
        const int m2 = nd_slots(Kb, batch, j, slots.data());
        if (m2 != m) {                                   // items join: every array to its new slots, the joining items' start values
            for (int s2 = 0, q = 0; s2 < m2; s2++) map[s2] = (q < m && prev[q] == slots[s2]) ? q++ : -1 - slots[s2];
            RTRY(cudaMemcpyAsync(L.dmap, map.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice, st));
            RTRY(cudaMemcpyAsync(L.dslots, slots.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice, st));
            for (int a = 0; a < narr; a++) {
                if (!m) { RTRY(ew_slot_gather<T>(nullptr, arr[a], L.dmap, m2, n, init[a], gout, kk, st)); continue; }   // start values only
                RTRY(ew_slot_gather<T>(arr[a], L.sc, L.dmap, m2, n, init[a], gout, kk, st));
                RTRY(cudaMemcpyAsync(arr[a], L.sc, (size_t)m2 * n * sizeof(T), cudaMemcpyDeviceToDevice, st));
            }
            m = m2; nm = n * m; prev.swap(slots);
        }
        const unsigned ge = ew_grid(nm);
        if (s == ND_PD) {
            for (int i = 0; i < npen; i++) {
                RTRY(pass((long long)j * npen + i, i));
                KernelSpan sp(KC_ELEMENTWISE, 1, st);
                k_pdv<T><<<ge, 256, 0, st>>>(L.a, npen, i, j > 0, L.sc, L.Sk, L.h, gY, nm);
                RTRY(cudaGetLastError());
            }
        } else {
            if (npen >= 2) {
                RTRY(pass(2LL * j + 1, 1));
                KernelSpan sp(KC_ELEMENTWISE, 1, st);
                k_pd2v<T><<<ge, 256, 0, st>>>(1, true, L.sc, gp, gq, L.h, gY, nm);
                RTRY(cudaGetLastError());
            }
            RTRY(pass(npen >= 2 ? 2LL * j : 0, 0));
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            k_pd2v<T><<<ge, 256, 0, st>>>(2, j > 0, L.sc, gp, gq, L.h, gY, nm);
            RTRY(cudaGetLastError());
        }
    }
    return cudaSuccess;
#undef RTRY
}

template <typename T>
cudaError_t nd_vjp_device(NdSolver s, const NdTerms& t, int npen, int maxIters, int iters, const void* tape, const T* gout, T* gY,
                          double* glam, void* ws, cudaStream_t st, int batch, const int* Kb) {
#define RTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
    const long long n = t.n;
    const int nb = batch > 0 ? batch : 1;
    if (glam) RTRY(cudaMemsetAsync(glam, 0, (size_t)nb * npen * sizeof(double), st));
    const int K = batch > 0 ? 0 : nd_K(s, maxIters, iters);
    if (n == 0 || (batch == 0 && K <= 0)) return cudaSuccess;
    NdVjpWs<T> L;
    nd_vjp_ws<T>(t, npen, glam != nullptr, (char*)ws, &L, batch);
    const char* tb = (const char*)tape + nd_tape_head_bytes(batch);
    if (s != ND_PDR) {
        RTRY(nd_vjp_items<T>(s, t, npen, nb, batch > 0 ? Kb : &K, tb, gout, gY, glam, L, st));
        if (batch > 0 && glam && s == ND_PD) {           // d/d of the penalties as given: PD_TV solved with npen lam_i
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            k_scale<<<ew_grid((long long)batch * npen), 256, 0, st>>>(glam, (long long)batch * npen, (double)npen);
            RTRY(cudaGetLastError());
        }
        return cudaSuccess;
    }
    const size_t sb = ptvv::vjp_tape_set_bytes(n);
    const unsigned ge = ew_grid(n);
    // the VJP of pass p (term i) for the upstream h into sc, and its edge gradients into glam[i]
    auto pass = [&](long long p, int i) -> cudaError_t {
        const FiberGeom& g = t.g[i];
        const uint32_t* F = (const uint32_t*)(tb + (size_t)p * 2 * sb);
        RTRY(ptvv::vjp_fibers_tape<T>(F, F + sb / 4, L.h, L.sc, L.gw, g.nf, g.len, g.inc, L.vscr, st));
        // one "image" of all edges: img_sums adds its sum to glam[2 * 0 + i]
        if (glam) RTRY(img_sums<T>(L.gw, g.nf * (long long)(g.len - 1), 1, L.scratch, nullptr, glam, i, 1.0, st));
        return cudaSuccess;
    };
    auto step = [&](bool start, int i, bool more) -> cudaError_t {
        KernelSpan sp(KC_ELEMENTWISE, 1, st);
        k_pdrv<T><<<ge, 256, 0, st>>>(L.a, npen, i, start, more, gout, L.sc, L.Sk, L.h, gY, n);
        return cudaGetLastError();
    };
    RTRY(step(true, npen - 1, K >= 2));
    for (int j = K - 2; j >= 0; j--)
        for (int i = 0; i < npen; i++) {
            RTRY(pass((long long)j * npen + i, i));
            RTRY(step(false, i, j > 0));
        }
    return cudaSuccess;
#undef RTRY
}

#define INST(T) \
    template cudaError_t pdr_tape_pass<T>(void*, long long, long long, const T*, FiberGeom, T, cudaStream_t); \
    template cudaError_t nd_tape_pass<T>(void*, long long, long long, const T*, FiberGeom, T, cudaStream_t, const T*, long long); \
    template size_t ws_bytes_nd_vjp<T>(const NdTerms&, int, bool, int); \
    template cudaError_t nd_vjp_device<T>(NdSolver, const NdTerms&, int, int, int, const void*, const T*, T*, double*, void*, cudaStream_t, \
                                          int, const int*); \
    template size_t ws_bytes_dr2_record<T>(size_t, size_t, int); \
    template size_t ws_bytes_dr2_vjp<T>(size_t, size_t, int); \
    template cudaError_t dr2_record_device<T>(size_t, size_t, int, int, const T*, T, T, T*, int, void*, void*, Engine, cudaStream_t); \
    template cudaError_t dr2_vjp_device<T>(size_t, size_t, int, int, int, const void*, const T*, T*, double*, void*, cudaStream_t); \
    template size_t ws_bytes_drw_record<T>(size_t, size_t, int); \
    template size_t ws_bytes_drw_vjp<T>(size_t, size_t, int); \
    template cudaError_t drw_record_device<T>(size_t, size_t, int, int, const T*, const T*, const T*, T*, int, void*, void*, Engine, cudaStream_t); \
    template cudaError_t drw_vjp_device<T>(size_t, size_t, int, int, int, const void*, const T*, T*, T*, T*, void*, cudaStream_t);
INST(double)
INST(float)

}  // namespace ptv
