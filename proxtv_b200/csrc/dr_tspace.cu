// dr_tspace.cu -- Douglas-Rachford (DR2_TV) schedule with NO standalone transposes.
//
// The column pass works on the column-major image ("N-space", axis-0 fibers contiguous); the row pass works on a transposed
// copy ("T-space", axis-1 fibers contiguous).  Instead of transposing between the passes with separate kernels, each scan
// kernel writes its result twice from its fill phase: once densely in its own space (that row is also the kernel's sparse
// value store) and once TRANSPOSED into the other space (8-byte writes one sector apart; the CTAs of the neighbouring
// fibers complete each sector and L2 merges them before they reach HBM).  One iteration = exactly two kernels:
//
//   cols (N-space):  stage t by TMA            -> s  = 2 (t - prox(t)) - t        dense: s (N)      transposed: sT (T)
//   rows (T-space):  stage YT - sT             -> t' = 0.5 (tT + 2 (YT - (in - prox(in))) - sT)
//                                                                                 dense: tT' (T)    transposed: t' (N)
//
// Y is transposed once per solve (YT).  Arithmetic, operation order and pass order are exactly those of the serial
// schedule (src/TV2Dopt.cpp:403-430); only where results are stored differs.  Works for a batch of images.
#include "ptv_internal.h"
#include "chunk_core.cuh"
#include <stdio.h>

namespace ptv {

template <typename T>
cudaError_t prox_fibers_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                       const T* lamv, cudaStream_t st, T* X2 = nullptr, long long inc2 = 0,
                                       const T* lamf = nullptr, long long fpi = 1);
template <typename T> cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st);
template <typename T> cudaError_t scatter_fibers(const T* in, T* X, FiberGeom g, cudaStream_t st);

static inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

template <typename T> size_t ws_arrays_dr2_tspace() { return 7; }

// returns 0 ok, 1 CUDA error, 2 shape not supported by the chunked kernel (nothing enqueued that matters: caller falls back)
template <typename T>
int dr2_tspace_body(size_t M, size_t N, int batch, const T* Y, T w1, T w2, T* out, int maxit, void* ws, double* scratch,
                    cudaStream_t st, bool plain_transposes) {
    const long long per = (long long)M * N, n = per * batch;
    char* w = (char*)ws; const size_t ab = al256((size_t)n * sizeof(T));
    T* t = (T*)w; w += ab; T* t2 = (T*)w; w += ab; T* tT = (T*)w; w += ab; T* tT2 = (T*)w; w += ab;
    T* s = (T*)w; w += ab; T* sT = (T*)w; w += ab; T* YT = (T*)w; w += ab;
    const FiberGeom gcols{(long long)N * batch, (int)M, 1};       // N-space: columns are contiguous fibers of length M
    const FiberGeom grows{(long long)M * batch, (int)N, 1};       // T-space: rows are contiguous fibers of length N
    const FiberGeom gstr{(long long)M * batch, (int)N, (long long)M};   // the rows as they lie in N-space (for the one-off transpose)
#define TTRY(expr) do { cudaError_t e__ = (expr); if (e__ == cudaErrorInvalidConfiguration) { cudaGetLastError(); return 2; } \
    if (e__ != cudaSuccess) { fprintf(stderr, "proxtv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); return 1; } } while (0)
    { KernelSpan sp(KC_ELEMENTWISE, 1, st); TTRY(gather_fibers<T>(Y, nullptr, IN_A, YT, gstr, st)); }             // YT, once
    TTRY(ew_image_means_x2<T>(Y, per, batch, t, scratch, st));                                                      // t = 2 mean
    TTRY(cudaMemcpyAsync(tT, t, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));                             // constant: same in T-space
    for (int it = 0; it <= maxit; it++) {
        const bool final = it == maxit;
        if (it == 0 && maxit > 0) {
            // constant first image: one fiber per image is solved and broadcast, directly into T-space
            TTRY(prox_const_fibers<T>(t, per, batch, (int)M, w1, s, st));
            TTRY(ew_dr_reflect_bcast<T>(tT, s, sT, n, per, (int)M, (long long)N, st));
        } else {
            { KernelSpan sp(KC_PROX_CONTIG, 1, st);
              TTRY(prox_fibers_chunked_contig<T>(t, nullptr, nullptr, IN_A, s, final ? OUT_DIFF : OUT_REFLECT, gcols, w1, nullptr, st,
                                                 plain_transposes ? nullptr : sT, (long long)N)); }
            if (plain_transposes) { KernelSpan sp(KC_ELEMENTWISE, 1, st); TTRY(gather_fibers<T>(s, nullptr, IN_A, sT, gstr, st)); }
        }
        if (plain_transposes) {
            // the fused row kernel stays in T-space (reads YT, sT, tT; writes tT'); one plain transpose brings t' back
            T* dstT = tT2;
            { KernelSpan sp(KC_PROX_STRIDED, 1, st);
              TTRY(prox_fibers_chunked_contig<T>(YT, sT, final ? nullptr : tT, IN_A_MINUS_B, dstT, final ? OUT_DR_ROWS_FINAL : OUT_DR_ROWS,
                                                 grows, w2, nullptr, st)); }
            { KernelSpan sp(KC_ELEMENTWISE, 1, st); TTRY(scatter_fibers<T>(dstT, final ? out : t2, gstr, st)); }
            if (!final) { T* tmp = t; t = t2; t2 = tmp; tmp = tT; tT = tT2; tT2 = tmp; }
            continue;
        }
        KernelSpan sp(KC_PROX_STRIDED, 1, st);
        if (!final) {
            TTRY(prox_fibers_chunked_contig<T>(YT, sT, tT, IN_A_MINUS_B, tT2, OUT_DR_ROWS, grows, w2, nullptr, st, t2, (long long)M));
            T* tmp = t; t = t2; t2 = tmp; tmp = tT; tT = tT2; tT2 = tmp;
        } else {
            TTRY(prox_fibers_chunked_contig<T>(YT, sT, nullptr, IN_A_MINUS_B, tT2, OUT_DR_ROWS_FINAL, grows, w2, nullptr, st, out, (long long)M));
        }
    }
#undef TTRY
    return 0;
}

template size_t ws_arrays_dr2_tspace<double>();
template size_t ws_arrays_dr2_tspace<float>();
template int dr2_tspace_body<double>(size_t, size_t, int, const double*, double, double, double*, int, void*, double*, cudaStream_t, bool);
template int dr2_tspace_body<float>(size_t, size_t, int, const float*, float, float, float*, int, void*, double*, cudaStream_t, bool);

}  // namespace ptv
