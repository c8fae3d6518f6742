// prox_dispatch.cu -- chooses the kernel family for one batched 1D prox over the fibers of an array.
//
//   contiguous fibers (inc == 1), len >= 64, fits shared memory  -> chunked speculative kernel, TMA staged
//   strided fibers, with scratch (default)                        -> tiled gather (fused input op) + chunked kernel + tiled scatter (fused output form)
//   strided fibers, ENGINE_CHUNKED_STRIDED or no scratch          -> chunked kernel staging FPB adjacent fibers directly
//   everything else (tiny fibers, weighted strided, ENGINE_SEQ)   -> sequential lane-per-fiber kernel
//
// With a per-fiber penalty table (prox_fibers_lamf: fiber j's penalty is lamf[j / fpi]) the lane engine (its per-lane instantiation,
// only for a table whose entries are all > 0, as the uniform route needs lam > 0), the chunked kernels (contiguous, and behind the
// gather -> scan -> scatter route) and the sequential kernel take the table.  Two routes decline it and pass the fibers down: the
// direct strided kernel of ENGINE_CHUNKED_STRIDED (to the gather route, or the sequential kernel without scratch) and the long-fiber
// tiles (to the sequential kernel).  Every fiber's result is the uniform pass's with its own penalty on the kernel family that ran it.
#include "ptv_internal.h"
#include "chunk_core.cuh"

namespace ptv {

template <typename T>
cudaError_t prox_fibers_seq(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv,
                            const int* list, long long nlist, cudaStream_t st, const T* lamf = nullptr, long long fpi = 1);
template <typename T>
cudaError_t prox_fibers_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                       const T* lamv, cudaStream_t st, T* X2 = nullptr, long long inc2 = 0,
                                       const T* lamf = nullptr, long long fpi = 1);
template <typename T>
cudaError_t prox_fibers_chunked_strided(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, T* V,
                                        cudaStream_t st);
template <typename T>
cudaError_t prox_long_fibers(const T* A, const T* B, InOp op, T* X, int out_op, FiberGeom g, T lam, T* scratch, long long scratch_elems,
                             cudaStream_t st);
long long lf_scratch_elems(long long nf, long long len);
template <typename T> cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st);
template <typename T> cudaError_t scatter_fibers(const T* in, T* X, FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_ex(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t prox_fibers_chunked_contig_sparse(const T* A, const T* B, InOp op, T* X, FiberGeom g, T lam, const T* lamv, uint32_t* Mk, T* Cv,
                                              cudaStream_t st, const T* lamf = nullptr, long long fpi = 1);
template <typename T>
cudaError_t scatter_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                  FiberGeom g, cudaStream_t st);
// elements of scratch the strided route needs for its sparse form: two staging arrays + per-chunk masks and entering values
long long strided_scratch_elems(long long nf, long long len) { return 2 * nf * len + 2 * nf * ((len + 31) / 32) + 64; }

// outcome of the long-fiber tiles per device, for tests (long_fiber_last in ptv_internal.h); stored + 2, so a slot never written reads -1
static int g_lf_last_d[MAX_DEVICES] = {};
void long_fiber_note(int v) { const int d = device_slot(); if (d >= 0) g_lf_last_d[d] = v + 2; }
int long_fiber_last() { const int d = device_slot(); const int v = d < 0 ? 0 : g_lf_last_d[d]; return v ? v - 2 : -1; }

template <typename T>
cudaError_t prox_fibers_ex(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv,
                           Engine eng, T* scratch, cudaStream_t st, long long scratch_elems, const T* lamf, long long fpi, bool lamf_pos) {
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    // plain unweighted prox over many fibers: the lane-per-fiber streaming engine (kernels_lane.cu), when the shape suits TMA tiling
    // and there are enough fibers to fill the machine without cutting them (a single long fiber stays with the chunked kernels,
    // which are also the bit-faithful ones behind the 1D entry points)
    if ((eng == ENGINE_AUTO || eng == ENGINE_LANE || eng == ENGINE_LANE_T) && op == IN_A && out_op == OUT_X && !lamv && (lamf ? lamf_pos : lam > T(0)) && g.len >= 64 && g.nf >= 1024) {
        const void* ptrs[2] = {A, X};
        if (ptvl::lane_shape_ok(g.nf, g.len, g.inc, sizeof(T), ptrs, 2)) {
            void* lscr = ptvl::lane_scratch(g.nf, g.len);
            if (lscr) {
                KernelSpan span(g.inc == 1 ? KC_PROX_CONTIG : KC_PROX_STRIDED, 1, st);
                cudaError_t e = ptvl::lane_prox<T>(ptvl::LANE_PLAIN, A, nullptr, nullptr, X, g.nf, g.len, g.inc, lam, lscr, st, nullptr, lamf, fpi);
                if (e != cudaErrorInvalidConfiguration) return e;
                cudaGetLastError(); span.cancel();
            }
        }
    }
    if (eng != ENGINE_SEQ && g.len >= 2 * 32) {
        if (g.inc == 1) {
            KernelSpan span(KC_PROX_CONTIG, 1, st);
            cudaError_t e = prox_fibers_chunked_contig<T>(A, B, C, op, X, out_op, g, lam, lamv, st, nullptr, 0, lamf, fpi);
            if (e != cudaErrorInvalidConfiguration) return e;
            cudaGetLastError();
            span.cancel();                  // refused before launching: the launch counters count kernels that ran
            // too long for shared memory: overlapping tiles, verified stitching (long_fiber.cu); the scratch convention for
            // this case is lf_scratch_elems() elements, which the 1D host entry points provide
            // (plain results only: the agreement test of the stitching compares prox values, which the fused output forms would hide)
            if (!lamv && !lamf && out_op == OUT_X && scratch && scratch_elems >= lf_scratch_elems(g.nf, g.len)) {
                KernelSpan lspan(KC_PROX_CONTIG, 1, st);
                e = prox_long_fibers<T>(A, B, op, X, out_op, g, lam, scratch, lf_scratch_elems(g.nf, g.len), st);
                if (e == cudaSuccess || e == cudaErrorNotReady) long_fiber_note(e == cudaSuccess ? 1 : 0);
                if (e == cudaSuccess) return e;
                if (e != cudaErrorInvalidConfiguration && e != cudaErrorNotReady) return e;
                if (e == cudaErrorInvalidConfiguration) lspan.cancel();      // NotReady: the tiles ran, their check failed
                cudaGetLastError();
            }
        } else if (!lamv) {
            // Strided fibers.  Default: tiled gather (input op fused) -> contiguous chunked kernel -> tiled scatter (output form
            // fused).  The scan is compute bound (IPC-limited, ~35 us of HBM time per 225 us pass), so the two extra streaming
            // kernels cost less than staging strided fibers directly at one CTA per SM; ENGINE_CHUNKED_STRIDED selects the
            // direct kernel (no transposed copy, FPB adjacent fibers per CTA) for comparison and for callers without scratch.
            const bool direct = (eng == ENGINE_CHUNKED_STRIDED) || !scratch || g.nf % g.inc != 0;
            if (direct && !lamf) {
                KernelSpan span(KC_PROX_STRIDED, 1, st);
                cudaError_t e = prox_fibers_chunked_strided<T>(A, B, C, op, X, out_op, g, lam,
                                                               (scratch && eng == ENGINE_CHUNKED_STRIDED) ? scratch : nullptr, st);
                if (e != cudaErrorInvalidConfiguration) return e;
                cudaGetLastError();
                span.cancel();
            }
            if (scratch && g.nf % g.inc == 0) {
                const long long n = g.nf * (long long)g.len;
                T* t1 = scratch; T* t2 = scratch + n;
                const FiberGeom gc{g.nf, g.len, 1};
                cudaError_t e;
                { KernelSpan span(KC_ELEMENTWISE, 1, st); e = gather_fibers<T>(A, B, op, t1, g, st); }
                if (e != cudaSuccess) return e;
                // with enough scratch the scan leaves a sparse result (no fill phase) and the scatter expands it while it transposes
                const bool sparse = scratch_elems >= strided_scratch_elems(g.nf, g.len);
                const long long lpf = ((long long)g.len + 31) / 32;
                T* Cv = scratch + 2 * n; uint32_t* Mk = reinterpret_cast<uint32_t*>(Cv + g.nf * lpf);
                { KernelSpan span(KC_PROX_STRIDED, 1, st);
                  // the gathered row of fiber j is row j: the penalty table applies unchanged
                  e = sparse ? prox_fibers_chunked_contig_sparse<T>(t1, nullptr, IN_A, t2, gc, lam, nullptr, Mk, Cv, st, lamf, fpi)
                             : prox_fibers_chunked_contig<T>(t1, nullptr, nullptr, IN_A, t2, OUT_X, gc, lam, nullptr, st, nullptr, 0, lamf, fpi);
                  if (e == cudaErrorInvalidConfiguration) span.cancel(); }
                if (e == cudaSuccess) {
                    KernelSpan span(KC_ELEMENTWISE, 1, st);
                    if (sparse) return out_op == OUT_X ? scatter_fibers_sparse<T>(t2, Mk, Cv, nullptr, nullptr, nullptr, IN_A, OUT_X, X, g, st)
                                                       : scatter_fibers_sparse<T>(t2, Mk, Cv, A, B, C, op, out_op, X, g, st);
                    return out_op == OUT_X ? scatter_fibers<T>(t2, X, g, st) : scatter_fibers_ex<T>(t2, A, B, C, op, out_op, X, g, st);
                }
                if (e != cudaErrorInvalidConfiguration) return e;
                cudaGetLastError();
            }
        }
    }
    KernelSpan span(g.inc == 1 ? KC_PROX_CONTIG : KC_PROX_STRIDED, 1, st);
    return prox_fibers_seq<T>(A, B, C, op, X, out_op, g, lam, lamv, nullptr, 0, st, lamf, fpi);
}

template <typename T>
cudaError_t prox_fibers_lamf(const T* A, const T* B, InOp op, T* X, FiberGeom g, const T* lamf, long long fpi, bool pos, Engine eng, T* scratch,
                             cudaStream_t st, long long scratch_elems) {
    return prox_fibers_ex<T>(A, B, nullptr, op, X, OUT_X, g, T(0), nullptr, eng, scratch, st, scratch_elems, lamf, fpi, pos);
}

template <typename T>
cudaError_t prox_fibers(const T* A, const T* B, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv, Engine eng,
                        T* scratch, cudaStream_t st, long long scratch_elems) {
    return prox_fibers_ex<T>(A, B, nullptr, op, X, out_op, g, lam, lamv, eng, scratch, st, scratch_elems);
}

#define INST(T) \
    template cudaError_t prox_fibers_ex<T>(const T*, const T*, const T*, InOp, T*, int, FiberGeom, T, const T*, Engine, T*, cudaStream_t, long long, \
                                           const T*, long long, bool); \
    template cudaError_t prox_fibers_lamf<T>(const T*, const T*, InOp, T*, FiberGeom, const T*, long long, bool, Engine, T*, cudaStream_t, long long); \
    template cudaError_t prox_fibers<T>(const T*, const T*, InOp, T*, int, FiberGeom, T, const T*, Engine, T*, cudaStream_t, long long);
INST(double)
INST(float)

}  // namespace ptv
