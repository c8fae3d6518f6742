// solver.cu -- device-resident outer loops: Douglas-Rachford (DR2_TV) and proximal Dykstra (PD2_TV, PD_TV).
//
// Semantics follow the reference exactly (same initialisation, pass order, iteration structure, stop test and info[]):
//   DR2_TV  src/TV2Dopt.cpp:352-444     PD2_TV  src/TV2Dopt.cpp:59-302     PD_TV  src/TVNDopt.cpp:48-252
// The reference's fixed 35 DR iterations are NOT a converged solve and the result depends on the pass order, so nothing
// here may be "improved" (SURVEY.md section 0.3).  All arrays stay in HBM for the whole solve; the only host round trip
// is the 8-byte stop criterion of the Dykstra loops, once per iteration.
#include "ptv_internal.h"
#include "chunk_core.cuh"
#include <float.h>
#include <limits.h>
#include <stdio.h>
#include <string.h>
#include <vector>

namespace ptv {

static inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static constexpr size_t SCRATCH_BYTES = (REDUCE_BLOCKS + 8) * sizeof(double);

#define PTV_TRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
    fprintf(stderr, "proxtv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); \
    if (info) info[INFO_RC] = RC_ERROR; return 0; } } while (0)

// ------------------------------------------------------------------------------------------------------------------
// Pipelined Douglas-Rachford iteration for one large column-major image.  The scan kernels are compute bound and the two
// tiled transposes around the row pass are HBM bound, so they are overlapped: each pass is issued as two half-kernels on two
// compute streams, and the transpose of a half starts on a third stream as soon as that half is done:
//     columns:  A(cols 0..N/2) | A(cols N/2..N)            gather(cols 0..N/2) runs under the second half of A
//     rows:     P(rows 0..M/2) | P(rows M/2..M)            scatter+combine(rows 0..M/2) runs under the second half of P
// Same kernels, same arithmetic, same results as the serial schedule; only the order of independent work changes.
template <typename T>
cudaError_t prox_fibers_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                       const T* lamv, cudaStream_t st, T* X2 = nullptr, long long inc2 = 0,
                                       const T* lamf = nullptr, long long fpi = 1);
template <typename T> cudaError_t gather_fibers_range(const T* A, const T* B, InOp op, T* out, FiberGeom g, int k_begin, int k_end, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_ex_range(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g,
                                    long long r_begin, long long r_end, cudaStream_t st);
template <typename T>
cudaError_t prox_fibers_chunked_contig_sparse(const T* A, const T* B, InOp op, T* X, FiberGeom g, T lam, const T* lamv, uint32_t* Mk, T* Cv,
                                              cudaStream_t st, const T* lamf = nullptr, long long fpi = 1);
template <typename T>
cudaError_t scatter_fibers_ex_sparse_range(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op,
                                           T* X, FiberGeom g, long long r_begin, long long r_end, cudaStream_t st);

struct DrPipe {
    static constexpr int MAXP = 8;
    cudaStream_t sa = nullptr, sb = nullptr, sx = nullptr, sg = nullptr;      // sg: origin stream of graph capture / replay
    cudaEvent_t e0 = nullptr, eG = nullptr, eS = nullptr, eIn = nullptr, eOut = nullptr, eA[MAXP] = {}, eP[MAXP] = {};
    // pieces each pass is cut into.  The overlap is close to zero-sum: the transposes saturate HBM and stretch the scans' memory
    // phases, so more pieces, or fewer scan CTAs per SM to make room for transpose CTAs, do not pay.
    int parts = 2;
    bool ok = false;
    bool init() {
        if (ok) return true;
        if (cudaStreamCreateWithFlags(&sa, cudaStreamNonBlocking) != cudaSuccess) return false;
        if (cudaStreamCreateWithFlags(&sb, cudaStreamNonBlocking) != cudaSuccess) return false;
        // the transpose stream gets the highest priority: its (small, memory-bound) CTAs must be dispatched ahead of the
        // still-pending CTAs of the next scan piece, otherwise they only run under that kernel's last wave
        int prio_least = 0, prio_greatest = 0;
        cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
        if (cudaStreamCreateWithPriority(&sx, cudaStreamNonBlocking, prio_greatest) != cudaSuccess) return false;
        if (cudaStreamCreateWithFlags(&sg, cudaStreamNonBlocking) != cudaSuccess) return false;
        cudaEvent_t* ev[] = {&e0, &eG, &eS, &eIn, &eOut};
        for (auto e : ev) if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) return false;
        for (int i = 0; i < MAXP; i++)
            if (cudaEventCreateWithFlags(&eA[i], cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&eP[i], cudaEventDisableTiming) != cudaSuccess) return false;
        return ok = true;
    }
};
// streams, events and the captured graph belong to one device: one set per device (calls are serialised by the C-ABI mutex)
static DrPipe g_pipe_d[MAX_DEVICES];
// the current device's set, ready; nullptr when it cannot be made or the device has no slot (the schedules that need it are then skipped)
static DrPipe* dev_pipe() { const int d = device_slot(); return d >= 0 && g_pipe_d[d].init() ? &g_pipe_d[d] : nullptr; }

// one iteration (or the final projection pair when `final`): t -> s (cols) -> x (rows); returns false on a CUDA error.
// Each pass is cut into p.parts pieces issued alternately on two compute streams; the transpose of a piece is queued on
// the high-priority stream as soon as that piece is done, so it runs under the following pieces.
template <typename T>
static bool dr_iteration_pipelined(DrPipe& p, size_t M, size_t N, const T* Y, T* t, T* s, T* x, T* scr, T w1, T w2, bool skip_cols,
                                   bool final, bool sparse, cudaStream_t st) {
    const long long n = (long long)M * N;
    T* t1 = scr; T* t2 = scr + n;
    // sparse row pass: the scan leaves segment values at their starts + per-chunk masks / entering values (third and fourth
    // staging arrays), and the fused scatter expands them while it transposes -- the scan kernel's fill phase is skipped
    const long long lpf = ((long long)N + 31) / 32;
    T* Cv = scr + 2 * n; uint32_t* Mk = reinterpret_cast<uint32_t*>(scr + 3 * n);
    const FiberGeom gr{(long long)M, (int)N, (long long)M};
    const int outA = final ? 2 : 1, outB = final ? 4 : 3;
    const int P = p.parts;
    auto cut = [](size_t len, int i, int parts) { return (long long)((len * (size_t)i / (size_t)parts) & ~(size_t)1); };
#define PCHK(e) do { if ((e) != cudaSuccess) return false; } while (0)
    PCHK(cudaEventRecord(p.e0, st));
    PCHK(cudaStreamWaitEvent(p.sa, p.e0, 0)); PCHK(cudaStreamWaitEvent(p.sb, p.e0, 0)); PCHK(cudaStreamWaitEvent(p.sx, p.e0, 0));
    for (int i = 0; i < P; i++) {
        cudaStream_t sc = (i & 1) ? p.sb : p.sa;
        const long long c0 = cut(N, i, P), c1 = (i + 1 == P) ? (long long)N : cut(N, i + 1, P);
        if (!skip_cols && c1 > c0) {
            KernelSpan sp(KC_PROX_CONTIG, 1, sc);
            PCHK(prox_fibers_chunked_contig<T>(t + c0 * (long long)M, nullptr, nullptr, IN_A, s + c0 * (long long)M, outA,
                                               FiberGeom{c1 - c0, (int)M, 1}, w1, nullptr, sc));
        }
        PCHK(cudaEventRecord(p.eA[i], sc));
        PCHK(cudaStreamWaitEvent(p.sx, p.eA[i], 0));
        if (c1 > c0) { KernelSpan sp(KC_ELEMENTWISE, 1, p.sx); PCHK(gather_fibers_range<T>(Y, s, IN_A_MINUS_B, t1, gr, (int)c0, (int)c1, p.sx)); }
    }
    PCHK(cudaEventRecord(p.eG, p.sx));
    PCHK(cudaStreamWaitEvent(p.sa, p.eG, 0)); PCHK(cudaStreamWaitEvent(p.sb, p.eG, 0));
    for (int j = 0; j < P; j++) {
        cudaStream_t sc = (j & 1) ? p.sb : p.sa;
        const long long r0 = cut(M, j, P), r1 = (j + 1 == P) ? (long long)M : cut(M, j + 1, P);
        if (r1 > r0) {
            KernelSpan sp(KC_PROX_STRIDED, 1, sc);
            if (sparse) PCHK(prox_fibers_chunked_contig_sparse<T>(t1 + r0 * (long long)N, nullptr, IN_A, t2 + r0 * (long long)N, FiberGeom{r1 - r0, (int)N, 1}, w2,
                                                                  nullptr, Mk + r0 * lpf, Cv + r0 * lpf, sc));
            else PCHK(prox_fibers_chunked_contig<T>(t1 + r0 * (long long)N, nullptr, nullptr, IN_A, t2 + r0 * (long long)N, 0,
                                                    FiberGeom{r1 - r0, (int)N, 1}, w2, nullptr, sc));
        }
        PCHK(cudaEventRecord(p.eP[j], sc));
        PCHK(cudaStreamWaitEvent(p.sx, p.eP[j], 0));
        if (r1 > r0) {
            KernelSpan sp(KC_ELEMENTWISE, 1, p.sx);
            if (sparse) PCHK(scatter_fibers_ex_sparse_range<T>(t2, Mk, Cv, Y, s, t, IN_A_MINUS_B, outB, x, gr, r0, r1, p.sx));
            else PCHK(scatter_fibers_ex_range<T>(t2, Y, s, t, IN_A_MINUS_B, outB, x, gr, r0, r1, p.sx));
        }
    }
    PCHK(cudaEventRecord(p.eS, p.sx));
    PCHK(cudaStreamWaitEvent(st, p.eS, 0));
#undef PCHK
    return true;
}

// the complete pipelined solve on origin stream st (plain launch order; also what gets captured into the CUDA graph)
template <typename T>
static int dr2_piped_body(size_t M, size_t N, const T* Y, T w1, T w2, T* out, int maxit, T* t, T* s, T* x, T* scr, double* scratch,
                          FiberGeom gc, long long n, bool sparse, cudaStream_t st) {
#define BTRY(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
    fprintf(stderr, "proxtv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); return 1; } } while (0)
    BTRY(ew_image_means_x2<T>(Y, (long long)M * N, 1, t, scratch, st));               // t = 2 mean      (:390-395)
    for (int it = 0; it <= maxit; it++) {
        const bool final = it == maxit, first = it == 0 && maxit > 0;
        if (first) {                                                      // constant first image: one fiber, broadcast
            BTRY(prox_const_fibers<T>(t, (long long)M * N, 1, (int)M, w1, x, st));
            BTRY(ew_dr_reflect_bcast<T>(t, x, s, n, (long long)M * N, gc.len, gc.inc, st));
        }
        if (!dr_iteration_pipelined<T>(*dev_pipe(), M, N, Y, t, s, final ? out : x, scr, w1, w2, first, final, sparse, st)) {
            BTRY(cudaGetLastError()); return 1; }
        if (!final) { T* tmp = t; t = x; x = tmp; }
    }
    return 0;
#undef BTRY
}

// ------------------------------------------------------------------------------------------------------------------
// lane_guard (declared in ptv_internal.h): is the lane engine a good choice for this data?
struct LaneGuardState { const void* y = nullptr; long long n = 0; double lam = 0.0; size_t ts = 0; int ok = -1; double* dev = nullptr; };
static LaneGuardState g_guard_d[MAX_DEVICES];
int lane_guard_last() { const int d = device_slot(); return d < 0 ? -1 : g_guard_d[d].ok; }
template <typename T>
Engine lane_guard(Engine eng, const T* y, long long n, double lam, cudaStream_t st) {
    if (eng != ENGINE_AUTO || n < 2 || !(lam > 0.0)) return eng;
    const int dev = device_slot();
    if (dev < 0) return ENGINE_CHUNKED;
    LaneGuardState& G = g_guard_d[dev];
    {   // evaluated on every call: the same buffer (the C ABI's own staging area, a caller's frame buffer) holds different data each time
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) { cudaGetLastError(); return eng; }
        if (!G.dev && cudaMalloc(&G.dev, 257 * sizeof(double)) != cudaSuccess) { cudaGetLastError(); G.dev = nullptr; return ENGINE_CHUNKED; }
        double step = 0.0;
        const long long ns = n < (1LL << 18) ? n : (1LL << 18);               // the first 256k elements: a few fibers' worth
        if (ew_mean_abs_step<T>(y, ns, G.dev, st) != cudaSuccess ||
            cudaMemcpyAsync(&step, G.dev, sizeof(double), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return ENGINE_CHUNKED; }
        const double kappa = sizeof(T) == 8 ? 1.0 : 2.0;                      // float32 windows hold twice the rows
        G.y = (const void*)y; G.n = n; G.lam = lam; G.ts = sizeof(T);
        G.ok = (step > 0.0 && lam <= kappa * step) ? 1 : 0;                   // a constant array (step == 0) is the lane engine's worst case
    }
    return G.ok ? eng : ENGINE_CHUNKED;
}
template Engine lane_guard<double>(Engine, const double*, long long, double, cudaStream_t);
template Engine lane_guard<float>(Engine, const float*, long long, double, cudaStream_t);

// ------------------------------------------------------------------------------------------------------------------
// Douglas-Rachford on the lane-per-fiber engine (kernels_lane.cu): two kernels per iteration, no transposed copies, 6 array
// sweeps per iteration (the algorithmic count, SURVEY.md 8d).  With x1 = prox_cols(t), x2 = prox_rows(Y - s):
//     columns   x1 = prox(t)                                    1 read + 1 write      CONTIG layout (TMA box in, TMA box out)
//     rows      s = 2 (t - x1) - t ; in = Y - s                 3 reads               STRIDED layout, formed in the feeder
//               t' = 0.5 (t + s + 2 x2) = (t - x1) + x2         1 write               formed in the drain
// (src/TV2Dopt.cpp:403-423; the last form is the reference's :419-422 with tb substituted, equal up to rounding), and the
// final projection pair (:427-430) s = t - x1 ; out = prox_rows(Y - s).  The first column pass sees the constant image
// 2 * mean, whose prox is that constant.
// ------------------------------------------------------------------------------------------------------------------
// Douglas-Rachford on the lane-per-fiber engine (kernels_lane.cu): two kernels per iteration, no transposed copies, 6 array
// sweeps per iteration (the algorithmic count, SURVEY.md 8d).  With x1 = prox_cols(t), x2 = prox_rows(Y - s):
//     columns   x1 = prox(t)                                    1 read + 1 write      CONTIG layout (TMA box in, TMA box out)
//     rows      s = 2 (t - x1) - t ; in = Y - s                 3 reads               STRIDED layout, formed in the feeder
//               t' = 0.5 (t + s + 2 x2) = (t - x1) + x2         1 write               formed in the drain
// (src/TV2Dopt.cpp:403-423; the last form is the reference's :419-422 with tb substituted, equal up to rounding), and the
// final projection pair (:427-430) s = t - x1 ; out = prox_rows(Y - s).  The first column pass sees the constant image
// 2 * mean, whose prox is that constant.
template <typename T>
static int dr2_lane_body(size_t M, size_t N, int batch, const T* Y, T w1, T w2, T* out, int maxit, T* t, T* t2, T* x1, double* scratch,
                         void* lscr, cudaStream_t st) {
#define LTRY(expr) do { cudaError_t e__ = (expr); if (e__ == cudaErrorInvalidConfiguration) { cudaGetLastError(); return 2; } \
    if (e__ != cudaSuccess) { fprintf(stderr, "proxtv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); return 1; } } while (0)
    LTRY(ew_image_means_x2<T>(Y, (long long)M * N, batch, t, scratch, st));                                   // t = 2 mean (:390-395)
    for (int it = 0; it <= maxit; it++) {
        const bool final = it == maxit, first = it == 0 && maxit > 0;
        // first half-iteration: prox_cols of the constant t is t itself, so the row pass takes t as x1 (d = t - t = 0 exactly)
        if (!first) { KernelSpan sp(KC_PROX_CONTIG, 1, st);
                      LTRY(ptvl::lane_prox<T>(ptvl::LANE_PLAIN, t, nullptr, nullptr, x1, (long long)N * batch, (int)M, 1, w1, lscr, st)); }
        { KernelSpan sp(KC_PROX_STRIDED, 1, st);
          LTRY(ptvl::lane_prox<T>(final ? ptvl::LANE_DR_B_FINAL : ptvl::LANE_DR_B, Y, first ? t : x1, t, final ? out : t2, (long long)M * batch,
                                  (int)N, (long long)M, w2, lscr, st)); }
        if (!final) { T* tmp = t; t = t2; t2 = tmp; }
    }
    return 0;
#undef LTRY
}

template <typename T> cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st);

// Lane-engine schedule of DR2_TV with BOTH passes as STRIDED lane passes (32 adjacent fibers = one contiguous line per sample), for
// either storage order: the pass along axis 0 (the reference's "columns", first) runs over row-major arrays, the pass along axis 1
// over column-major arrays; every tile lands as it is, the Douglas-Rachford arithmetic sits in the drains, and each pass writes
// its results transposed into the other pass's layout (kernels_lane.cu: LOP_DRA / LOP_DRB):
//     axis-0 pass (Tr, Yr row-major):   x1 = prox(t) ; d = t - x1 ; u = Y - (2 d - t)   -> Uc, Dc (column-major)      (:405-411)
//     axis-1 pass (Uc, Dc col-major):   x2 = prox(u) ; t' = d + x2                     -> Tr (row-major)             (:415-422)
//     final:  u = Y - (t - x1) ; out = prox(u)                                                                       (:427-430)
// Same expressions, same association as the staged forms above: the two schedules agree bit for bit.  A row-major image (torch
// tensors, the batched entry points) needs no copy at all: Y is Yr and the last pass writes its result transposed; a column-major
// image (the reference's layout) is transposed once into Yr, and its first half-iteration -- the prox of the constant start image
// is that constant -- is a plain elementwise kernel.
template <typename T>
static int dr2_lane_t_body(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit, T* Tr, T* Yr_buf, T* Uc, T* Dc,
                           double* scratch, void* lscr, cudaStream_t st) {
#define LTRY(expr) do { cudaError_t e__ = (expr); if (e__ == cudaErrorInvalidConfiguration) { cudaGetLastError(); return 2; } \
    if (e__ != cudaSuccess) { fprintf(stderr, "proxtv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); return 1; } } while (0)
    const long long n = (long long)M * N * batch;
    const long long nf0 = (long long)N * batch, nf1 = (long long)M * batch;           // fibers along axis 0 (length M), along axis 1 (length N)
    const T* Yr = row_major ? Y : Yr_buf;
    LTRY(ew_image_means_x2<T>(Y, (long long)M * N, batch, Tr, scratch, st));         // t = 2 mean (:390-395): constant, so layout-free
    // One transposition per solve.  Column-major input: Yr = every image transposed.  Row-major input: the first half-iteration
    // needs Y in column-major order once (u = Y - (2 (t - t) - t) with the constant start image t; a lane pass over constant fibers
    // would be its worst case: not a single break, every fiber through the repair path); it is gathered into Dc and turned into
    // (Uc, Dc) in place.
    bool first_done = false;
    if (!row_major) {
        if (maxit > 0) { LTRY(ew_dr_first<T>(Y, Tr, Uc, Dc, n, st)); first_done = true; }
        KernelSpan sp(KC_ELEMENTWISE, 1, st);
        LTRY(gather_fibers<T>(Y, nullptr, IN_A, Yr_buf, FiberGeom{nf1, (int)N, (long long)M}, st));
    } else if (maxit > 0) {
        { KernelSpan sp(KC_ELEMENTWISE, 1, st);
          LTRY(gather_fibers<T>(Y, nullptr, IN_A, Dc, FiberGeom{nf0, (int)M, (long long)N}, st)); }
        LTRY(ew_dr_first<T>(Dc, Tr, Uc, Dc, n, st)); first_done = true;
    }
    for (int it = 0; it <= maxit; it++) {
        const bool final = it == maxit;
        if (!(it == 0 && first_done)) { KernelSpan sp(KC_PROX_CONTIG, 1, st);
            LTRY(ptvl::lane_prox<T>(final ? ptvl::LANE_DRA_FINAL : ptvl::LANE_DRA, Tr, Yr, Tr, Uc, nf0, (int)M, (long long)N, w1, lscr, st, Dc)); }
        { KernelSpan sp(KC_PROX_STRIDED, 1, st);
          if (final) LTRY(ptvl::lane_prox<T>(row_major ? ptvl::LANE_PLAIN_T : ptvl::LANE_PLAIN, Uc, nullptr, nullptr, out, nf1, (int)N, (long long)M, w2, lscr, st));
          else LTRY(ptvl::lane_prox<T>(ptvl::LANE_DRB, Uc, Dc, nullptr, Tr, nf1, (int)N, (long long)M, w2, lscr, st)); }
    }
    return 0;
#undef LTRY
}

template <typename T>
int dr2_tspace_body(size_t M, size_t N, int batch, const T* Y, T w1, T w2, T* out, int maxit, void* ws, double* scratch, cudaStream_t st,
                    bool plain_transposes);

// aux, aux_gen: the lane engine's scratch and its allocation count -- a regrown scratch can reuse the address with another layout
// (records after a larger counter region), which the kernel arguments baked into the graph would not follow
struct DrGraphKey {
    size_t tsize, M, N; const void* Y; void* out; void* ws; double w1, w2; int maxit; const void* aux; unsigned long long aux_gen;
    bool operator==(const DrGraphKey& o) const {
        return tsize == o.tsize && M == o.M && N == o.N && Y == o.Y && out == o.out && ws == o.ws && w1 == o.w1 && w2 == o.w2 &&
               maxit == o.maxit && aux == o.aux && aux_gen == o.aux_gen;
    }
};
struct DrGraph { cudaGraphExec_t exec = nullptr; DrGraphKey key{}; long long launches[KC_COUNT] = {0, 0, 0}; };
static DrGraph g_dr_graph_d[MAX_DEVICES];

// ------------------------------------------------------------------------------------------------------------------
template <typename T> size_t ws_bytes_dr2(size_t M, size_t N, int batch) {
    size_t n = M * N * (size_t)batch;
    return 7 * align256(n * sizeof(T)) + SCRATCH_BYTES;      // plain schedule: t, s, x, 2 staging; T-space schedule: 7 arrays
}

template <typename T>
int dr2_lane_pick(size_t M, size_t N, int batch, int row_major, const T* Y, const T* out, const void* ws, T w1, T w2, Engine eng,
                  void** lscr) {
    *lscr = nullptr;
    const void* lane_ptrs[3] = {Y, out, ws};
    const bool lane_t = eng == ENGINE_LANE_T || row_major;
    bool lane = (eng == ENGINE_AUTO || eng == ENGINE_LANE || eng == ENGINE_LANE_T) && w1 > T(0) && w2 > T(0) && M >= 2 && N >= 2 && dev_pipe() &&
                ptvl::lane_shape_ok((long long)N * batch, (int)M, lane_t ? (long long)N : 1, sizeof(T), lane_ptrs, 3) &&
                ptvl::lane_shape_ok((long long)M * batch, (int)N, (long long)M, sizeof(T), lane_ptrs, 3) &&
                (!lane_t || (((long long)M * sizeof(T)) % 16 == 0 && ((long long)N * sizeof(T)) % 16 == 0));
    if (lane) {
        void* a1 = ptvl::lane_scratch((long long)N * batch, (int)M); void* a2 = ptvl::lane_scratch((long long)M * batch, (int)N);
        *lscr = a2; lane = a1 && a2;                // the second call returns the (possibly grown) buffer both passes use
    }
    return lane ? (lane_t ? 2 : 1) : 0;
}

template <typename T>
int dr2_device(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit, double* info, void* ws,
               Engine eng, cudaStream_t st) {
    const long long n = (long long)M * (long long)N * batch;
    if (n == 0) { if (info) { info[INFO_ITERS] = 0; info[INFO_RC] = RC_OK; } return 0; }
    char* w = (char*)ws;
    T* t = (T*)w; w += align256(n * sizeof(T));
    T* s = (T*)w; w += align256(n * sizeof(T));
    T* x = (T*)w; w += align256(n * sizeof(T));
    T* scr = (T*)w; w += 4 * align256(n * sizeof(T));      // gather/scatter staging of the strided pass (+2 arrays of the T-space schedule)
    double* scratch = (double*)w;
    if (maxit <= 0) maxit = MAX_ITERS_DR;                                     // TV2Dopt.cpp:387
    eng = lane_guard<T>(eng, Y, n, (double)(w1 > w2 ? w1 : w2), st);        // AUTO: the lane engine only while segments stay short
    // first pass: fibers along axis 0 (length M); second pass: along axis 1 (length N) -- the order is part of the contract.
    // column-major: axis-0 fibers are contiguous, axis-1 fibers have stride M; row-major storage swaps the two roles.
    const FiberGeom gc = row_major ? FiberGeom{(long long)N * batch, (int)M, (long long)N} : FiberGeom{(long long)N * batch, (int)M, 1};
    const FiberGeom gr = row_major ? FiberGeom{(long long)M * batch, (int)N, 1} : FiberGeom{(long long)M * batch, (int)N, (long long)M};
    // Schedule.  AUTO (and ENGINE_PIPELINED): for a large single column-major image the gather/scatter schedule with the
    // transposes issued on a separate high-priority stream; ENGINE_TSPACE: the transposeless T-space schedule (dr_tspace.cu: two
    // kernels per iteration, each writing its result in both layouts -- kept for comparison); everything else: the plain serial schedule below.
    // The whole solve is captured once into a CUDA graph and replayed while the call's arguments stay the same (no host
    // launch latency); event timing of single launches needs plain launches, so profiling bypasses the graph.
    const bool tpose = eng == ENGINE_TPOSE;
    const bool tspace = (eng == ENGINE_TSPACE || tpose) && !row_major && M >= 64 && N >= 64 && dev_pipe();
    const bool piped = (eng == ENGINE_AUTO || eng == ENGINE_PIPELINED) && !row_major && batch == 1 && M >= 1024 && N >= 1024 && M % 2 == 0 && N % 2 == 0 &&
                       (size_t)((M > N ? M : N) * sizeof(T)) <= 96 * 1024 && dev_pipe();
    // lane-per-fiber engine: images whose row pitch suits TMA tiling, positive weights.  Column-major: the staged schedule (column
    // pass over contiguous fibers) or, engine lane-t, the transposed one; row-major: only the transposed schedule applies.
    void* lscr = nullptr;
    const int lane_sched = dr2_lane_pick<T>(M, N, batch, row_major, Y, out, ws, w1, w2, eng, &lscr);
    const bool lane = lane_sched != 0, lane_t = lane_sched == 2;
    if (lane || tspace || piped) {
        auto body = [&](cudaStream_t bs) -> int {
            if (lane) return lane_t ? dr2_lane_t_body<T>(M, N, batch, row_major, Y, w1, w2, out, maxit, t, s, x, scr, scratch, lscr, bs)
                                   : dr2_lane_body<T>(M, N, batch, Y, w1, w2, out, maxit, t, s, x, scratch, lscr, bs);
            return tspace ? dr2_tspace_body<T>(M, N, batch, Y, w1, w2, out, maxit, ws, scratch, bs, tpose)
                          : dr2_piped_body<T>(M, N, Y, w1, w2, out, maxit, t, s, x, scr, scratch, gc, n, eng == ENGINE_AUTO && sizeof(T) == 8, bs);
        };
        DrGraphKey key{sizeof(T) + (tspace ? 100u : 0u) + (tpose ? 200u : 0u) + (eng == ENGINE_AUTO ? 400u : 0u) + (lane ? 800u : 0u) + (lane && lane_t ? 50u : 0u) + (row_major ? 25u : 0u) + 1000u * (size_t)batch, M, N, (const void*)Y, (void*)out, ws, (double)w1,
                       (double)w2, maxit, lane ? lscr : nullptr, lane ? ptvl::lane_scratch_generation() : 0ull};
        int rc = -1;
        if (!profile_is_enabled()) {
            DrPipe& P = *dev_pipe();                        // every schedule here took it, so the device has a slot
            DrGraph& G = g_dr_graph_d[device_slot()];
            if (!(G.exec && G.key == key)) {
                if (G.exec) { cudaGraphExecDestroy(G.exec); G.exec = nullptr; }
                long long c0[KC_COUNT], c1[KC_COUNT];
                profile_counters(c0);
                cudaGraph_t graph = nullptr;
                bool okc = cudaStreamBeginCapture(P.sg, cudaStreamCaptureModeRelaxed) == cudaSuccess;
                if (okc) {
                    rc = body(P.sg);
                    okc = (cudaStreamEndCapture(P.sg, &graph) == cudaSuccess) && rc == 0 && graph;
                }
                if (okc) okc = cudaGraphInstantiate(&G.exec, graph, 0) == cudaSuccess;
                if (graph) cudaGraphDestroy(graph);
                profile_counters(c1);
                for (int i = 0; i < KC_COUNT; i++) { G.launches[i] = c1[i] - c0[i]; c1[i] = -G.launches[i]; }
                profile_add(c1);                                              // the capture itself launched nothing
                if (!okc) { cudaGetLastError(); G.exec = nullptr; } else G.key = key;
            }
            if (G.exec) {
                PTV_TRY(cudaEventRecord(P.eIn, st));
                PTV_TRY(cudaStreamWaitEvent(P.sg, P.eIn, 0));
                PTV_TRY(cudaGraphLaunch(G.exec, P.sg));
                PTV_TRY(cudaEventRecord(P.eOut, P.sg));
                PTV_TRY(cudaStreamWaitEvent(st, P.eOut, 0));
                profile_add(G.launches);
                if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; }
                return 0;
            }
        }
        if (rc != 2) rc = body(st);              // 2: shape not supported by the chunked kernel (reported before anything ran)
        if (rc == 0) { if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; } return 0; }
        if (rc == 1) { if (info) info[INFO_RC] = RC_ERROR; return 0; }
        // rc == 2: fall through to the plain schedule
    }
    PTV_TRY(ew_image_means_x2<T>(Y, (long long)M * N, batch, t, scratch, st));        // :390-395
    for (int it = 0; it < maxit; it++) {                                      // :403-423
        if (it == 0 && eng != ENGINE_SEQ) {
            // the first input is the constant image 2*mean: every axis-0 fiber of an image is the same constant vector, so
            // one fiber per image is solved (same arithmetic, registers only) and broadcast -- identical result, and it
            // spares the chunked kernel its worst case (a fiber without a single break).
            PTV_TRY(prox_const_fibers<T>(t, (long long)M * N, batch, (int)M, w1, x, st));
            PTV_TRY(ew_dr_reflect_bcast<T>(t, x, s, n, (long long)M * N, gc.len, gc.inc, st));
        } else
        PTV_TRY(prox_fibers<T>(t, nullptr, IN_A, s, 1 /*reflect: s = 2(t - prox) - t*/, gc, w1, nullptr, eng, scr, st, 4 * n));
        // second half fused into the row pass: in = Y - s ; tb = Y - (in - prox) ; tb = 2 tb - s ; t' = 0.5 (t + tb)
        PTV_TRY(prox_fibers_ex<T>(Y, s, t, IN_A_MINUS_B, x, 3 /*OUT_DR_ROWS*/, gr, w2, nullptr, eng, scr, st, 4 * n));
        { T* tmp = t; t = x; x = tmp; }                                       // t' was written to x: ping-pong
    }
    PTV_TRY(prox_fibers<T>(t, nullptr, IN_A, s, 2 /*s = t - prox*/, gc, w1, nullptr, eng, scr, st, 4 * n));   // :427-430
    PTV_TRY(prox_fibers_ex<T>(Y, s, nullptr, IN_A_MINUS_B, out, 4 /*OUT_DR_ROWS_FINAL*/, gr, w2, nullptr, eng, scr, st, 4 * n));
    if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; }            // :433-436 (INFO_GAP is left untouched)
    return 0;                                                                 // :440 (the reference returns 0 on success)
}

// ------------------------------------------------------------------------------------------------------------------
// DR2L1W_TV (src/TV2DWopt.cpp:46-140): the Douglas-Rachford skeleton of DR2_TV with per-edge weights -- W1: (M-1) x N (column
// fibers), W2: M x (N-1) (row fibers), each with len - 1 samples per fiber under its pass's slicing rule -- and the opposite reflection
// signs (:115, :125).  `batch` images back to back, column-major or C order: the pass order (columns first) is the same, only the
// stride roles swap.  The strided pass (rows of column-major images, columns of C-ordered ones) goes through the same gather ->
// contiguous chunked kernel -> fused scatter route as DR2_TV, its weights gathered once; the contiguous pass runs the chunked kernel
// in place (DrwPasses).
template <typename T> cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                  FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t expand_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                 FiberGeom g, cudaStream_t st);

template <typename T>
cudaError_t DrwPasses<T>::init(size_t M, size_t N, int batch, int row_major, const T* W1, const T* W2, Engine e, void* stage, cudaStream_t st) {
    g[0] = row_major ? FiberGeom{(long long)N * batch, (int)M, (long long)N} : FiberGeom{(long long)N * batch, (int)M, 1};
    g[1] = row_major ? FiberGeom{(long long)M * batch, (int)N, 1} : FiberGeom{(long long)M * batch, (int)N, (long long)M};
    W[0] = M > 1 ? W1 : nullptr; W[1] = N > 1 ? W2 : nullptr;
    eng = e;
    const size_t ab = align256(M * N * (size_t)batch * sizeof(T));
    char* w = (char*)stage;
    t1 = (T*)w; t2 = (T*)(w + ab); wg = (T*)(w + 2 * ab); Cv = (T*)(w + 3 * ab);
    long long ncv = 0;                                        // per-chunk masks / entering values of the sparse results
    for (int a = 0; a < 2; a++) {
        fast[a] = eng != ENGINE_SEQ && g[a].len >= 64;
        const long long c = g[a].nf * (((long long)g[a].len + 31) / 32);
        if (fast[a] && c > ncv) ncv = c;
    }
    Mk = reinterpret_cast<uint32_t*>(Cv + ncv);
    // by storage order, not by stride: a column-major image with M == 1 keeps the row route it always had
    const int s = strided = row_major ? 0 : 1;
    if (fast[s]) { KernelSpan sp(KC_ELEMENTWISE, 1, st);
                   return gather_fibers<T>(W[s], nullptr, IN_A, wg, FiberGeom{g[s].nf, g[s].len - 1, g[s].inc}, st); }
    return cudaSuccess;
}

template <typename T>
cudaError_t DrwPasses<T>::run(int axis, const T* A, const T* B, const T* C, InOp op, T* X, int out_op, cudaStream_t st) {
    const FiberGeom& G = g[axis];
    const bool gathered = axis == strided;
    // contiguous pass, output forms the chunked kernel's fill knows: prox_fibers_ex (chunked kernel, else the sequential one)
    if (!gathered && out_op < OUT_DRW_ROWS) return prox_fibers_ex<T>(A, B, C, op, X, out_op, G, T(0), W[axis], eng, nullptr, st, 0);
    if (fast[axis]) {
        cudaError_t e;
        if (gathered) { KernelSpan sp(KC_ELEMENTWISE, 1, st); e = gather_fibers<T>(A, B, op, t1, G, st); if (e != cudaSuccess) return e; }
        { KernelSpan sp(gathered ? KC_PROX_STRIDED : KC_PROX_CONTIG, 1, st);
          e = gathered ? prox_fibers_chunked_contig_sparse<T>(t1, nullptr, IN_A, t2, FiberGeom{G.nf, G.len, 1}, T(0), wg, Mk, Cv, st)
                      : prox_fibers_chunked_contig_sparse<T>(A, B, op, t2, G, T(0), W[axis], Mk, Cv, st);      // no fill: expanded below
          if (e == cudaErrorInvalidConfiguration) sp.cancel(); }
        if (e == cudaErrorInvalidConfiguration) { cudaGetLastError(); fast[axis] = false; }
        else {
            if (e != cudaSuccess) return e;
            KernelSpan sp(KC_ELEMENTWISE, 1, st);
            const bool plain = out_op == OUT_X;               // the plain scatter never looks at the input
            return gathered ? scatter_fibers_sparse<T>(t2, Mk, Cv, plain ? nullptr : A, plain ? nullptr : B, plain ? nullptr : C, op, out_op, X, G, st)
                           : expand_fibers_sparse<T>(t2, Mk, Cv, A, B, C, op, out_op, X, G, st);
        }
    }
    return prox_fibers_ex<T>(A, B, C, op, X, out_op, G, T(0), W[axis], ENGINE_SEQ, nullptr, st, 0);
}

template <typename T>
int drw_device(size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit, double* info, void* ws,
               Engine eng, cudaStream_t st) {
    const long long n = (long long)M * (long long)N * batch;
    if (maxit <= 0) maxit = MAX_ITERS_DR;                                     // TV2DWopt.cpp:82
    if (n == 0) { if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; } return 0; }
    char* w = (char*)ws;
    T* t = (T*)w; w += align256(n * sizeof(T));
    T* s = (T*)w; w += align256(n * sizeof(T));
    T* x = (T*)w; w += align256(n * sizeof(T));
    DrwPasses<T> P;
    PTV_TRY(P.init(M, N, batch, row_major, W1, W2, eng, w, st));
    w += 4 * align256(n * sizeof(T));
    double* scratch = (double*)w;
    PTV_TRY(ew_image_means_x2<T>(Y, (long long)M * N, batch, t, scratch, st));   // :85-89
    for (int it = 0; it <= maxit; it++) {                                     // :94-119, then the final pair :122-125
        const bool final = it == maxit;
        // columns: s = 2 (t - prox_W1(t)) - t   (final: s = t - prox_W1(t))
        PTV_TRY(P.run(0, t, nullptr, nullptr, IN_A, s, final ? OUT_DIFF : OUT_REFLECT, st));
        // rows: in = Y - s ; tb = (in - prox_W2(in)) - Y ; tb = -2 tb - s ; t' = 0.5 (t + tb)   (final: out = -s - tb)
        PTV_TRY(P.run(1, Y, s, t, IN_A_MINUS_B, final ? out : x, final ? OUT_DRW_ROWS_FINAL : OUT_DRW_ROWS, st));
        if (!final) { T* tmp = t; t = x; x = tmp; }
    }
    if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; }            // :128-131
    return 0;                                                                 // :135 (returns 0 on success, like DR2_TV)
}

// ------------------------------------------------------------------------------------------------------------------
// batch >= 1: the single-item layout for the whole batch, then NdItems' arrays (NdItems::split)
template <typename T> size_t ws_bytes_pd(long long n, int npen, int batch) {
    if (batch > 0) return ws_bytes_pd<T>(n * batch, npen, 0) + align256((size_t)(n * batch) * sizeof(T)) +
                          align256((size_t)batch * REDUCE_BLOCKS * sizeof(double)) + align256((size_t)batch * sizeof(double)) +
                          align256((size_t)batch * sizeof(int)) + align256((size_t)batch * (npen > 0 ? npen : 1) * sizeof(T));
    int arrays = 2 * npen + 4;   // PD_TV: p_i, z_i + 3 staging ; PD2_TV (npen <= 2): p, q, z, xl + 3 staging
    if (arrays < 8) arrays = 8;
    return (size_t)arrays * align256((size_t)n * sizeof(T)) + SCRATCH_BYTES + align256(2 * 64 * sizeof(void*));
}

int nd_slots(const int* K, int batch, int j, int* slots) {
    int m = 0;
    for (int b = 0; b < batch; b++)
        if (K[b] > j) { if (slots) slots[m] = b; m++; }
    return m;
}

// The fibers of `items` items of one term's geometry g: an item is the slowest axis, so its fibers are a contiguous range
static FiberGeom items_geom(const FiberGeom& g, int items) { return FiberGeom{g.nf * items, g.len, g.inc}; }

// The items of a PD_TV / PD2_TV solve (DESIGN.md section 16); a single-item call is one item.  K[b] is INT_MAX while item b runs, then
// the iterations it ran; the running items sit in the slots nd_slots gives them, slots[0..m).  Each iteration's stop values come back in
// one read-back; an item that stops gets its info row and its x copied to its place in the output, and the others' state arrays move to
// their new slots through a staging array (the moves of one array overlap, so they cannot be made in place).
template <typename T> struct NdItems {
    int batch = 0, m = 0; long long n = 0; T* out = nullptr; double* info = nullptr;
    std::vector<int> K, slots, next, map; std::vector<double> stop;
    T* x = nullptr; double* partial = nullptr; double* dstop = nullptr; int* dmap = nullptr; T* dlam = nullptr;
    NdItems(int b, long long n_, T* out_, double* info_)
        : batch(b), m(b), n(n_), out(out_), info(info_), K(b, INT_MAX), slots(b), next(b), map(b), stop(b) {
        nd_slots(K.data(), b, 0, slots.data());
    }
    // The device arrays.  w: a batch's, the workspace past the single-item layout of the whole batch (ws_bytes_pd).  nullptr: one item,
    // which iterates in its output and reduces in the single-item layout's scratch and dres, so its workspace is the single-item one.
    void split(char* w, double* scratch, double* dres) {
        if (!w) { x = out; partial = scratch; dstop = dres; return; }
        const int b = batch;
        x = (T*)w; w += align256((size_t)(n * b) * sizeof(T));
        partial = (double*)w; w += align256((size_t)b * REDUCE_BLOCKS * sizeof(double));
        dstop = (double*)w; w += align256((size_t)b * sizeof(double));
        dmap = (int*)w; w += align256((size_t)b * sizeof(int));
        dlam = (T*)w;
    }
    void row(int b, int iters, double s) {
        info[3 * (size_t)b + INFO_ITERS] = iters; info[3 * (size_t)b + INFO_GAP] = s;
        info[3 * (size_t)b + INFO_RC] = iters >= MAX_ITERS_PD ? RC_ITERS : RC_OK;
    }
    // after `iters` iterations; go(stop) is the solver's loop condition for one item; arrays[0] is x
    template <class Go> cudaError_t step(int iters, Go go, T* const* arrays, int narr, T* stage, cudaStream_t st) {
        cudaError_t e = cudaMemcpyAsync(stop.data(), dstop, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return e;
        int gone = 0;
        for (int s = 0; s < m; s++) {
            if (go(stop[s])) continue;
            const int b = slots[s];
            K[b] = iters; row(b, iters, stop[s]); gone++;
            if (x + (size_t)s * n == out + (size_t)b * n) continue;
            e = cudaMemcpyAsync(out + (size_t)b * n, x + (size_t)s * n, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return e;
        }
        if (!gone) return cudaSuccess;
        const int m2 = nd_slots(K.data(), batch, iters, next.data());
        if (m2 > 0) {
            for (int s2 = 0, s = 0; s2 < m2; s2++) { while (slots[s] != next[s2]) s++; map[s2] = s; }    // both in increasing b
            e = cudaMemcpyAsync(dmap, map.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice, st);
            for (int a = 0; a < narr && e == cudaSuccess; a++) {
                e = ew_slot_gather<T>(arrays[a], stage, dmap, m2, n, 0, nullptr, T(0), st);
                if (e == cudaSuccess) e = cudaMemcpyAsync(arrays[a], stage, (size_t)m2 * n * sizeof(T), cudaMemcpyDeviceToDevice, st);
            }
            if (e != cudaSuccess) return e;
        }
        slots.swap(next); m = m2;
        return cudaSuccess;
    }
    // items that never ran (no elements, no terms)
    void rest(int iters) { for (int b = 0; b < batch; b++) if (K[b] == INT_MAX) row(b, iters, DBL_MAX); }
};

// The penalties of a PD_TV / PD2_TV solve, lam[b * stride + i] for item b and term i: stride 0, one row shared by every item; stride npen,
// one row per item (DESIGN.md section 16.1).  A pass over the running items takes the uniform kernels with scalar(i) when they all have
// the same penalty for term i, else the per-fiber kernels with table(i): their penalties in slot order, in the device table I.dlam
// ([npen][batch]), uploaded by sync() whenever the running items change -- before the first pass and after each compaction, in the
// stream order of the iteration's other work.
template <typename T> struct NdPens {
    const double* lam; int stride, npen, batch;
    std::vector<T> host; std::vector<char> uni, pos; int m = -1;
    NdPens(const double* l, int s, int np, int b) : lam(l), stride(s), npen(np), batch(b), host((size_t)np * b), uni(np, 1), pos(np, 0) {}
    T at(int b, int i) const { return (T)lam[(size_t)b * stride + i]; }
    // the largest penalty of the whole table (the lane guard's)
    double max() const {
        double v = 0.0;
        for (int b = 0; b < (stride ? batch : 1); b++) for (int i = 0; i < npen; i++) if (lam[(size_t)b * stride + i] > v) v = lam[(size_t)b * stride + i];
        return v;
    }
    cudaError_t sync(const NdItems<T>& I, cudaStream_t st) {
        if (!stride || I.m == m) return cudaSuccess;
        m = I.m;
        bool all = true;
        for (int i = 0; i < npen; i++) {
            T* h = host.data() + (size_t)i * batch;
            for (int s = 0; s < m; s++) h[s] = at(I.slots[s], i);
            uni[i] = 1; pos[i] = 1;
            for (int s = 1; s < m; s++) if (memcmp(&h[s], &h[0], sizeof(T))) { uni[i] = 0; break; }
            for (int s = 0; s < m; s++) if (!(h[s] > T(0))) { pos[i] = 0; break; }     // a zero keeps the table off the lane engine
            all = all && uni[i];
        }
        return all ? cudaSuccess : cudaMemcpyAsync(I.dlam, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    T scalar(int i) const { return stride ? host[(size_t)i * batch] : at(0, i); }
    const T* table(const NdItems<T>& I, int i) const { return stride && !uni[i] ? I.dlam + (size_t)i * batch : nullptr; }
};

// One prox pass of term i over the running items' fibers g (fpi fibers per item), with their penalties, and its tape pass p (tp set)
template <typename T>
static cudaError_t nd_pass(const T* A, const T* B, InOp op, T* X, FiberGeom g, long long fpi, const NdPens<T>& L, const NdItems<T>& I, int i,
                           Engine eng, T* scr, long long scr_elems, char* tp, long long nt, long long p, cudaStream_t st) {
    const T* lamf = L.table(I, i);
    cudaError_t e = lamf ? prox_fibers_lamf<T>(A, B, op, X, g, lamf, fpi, L.pos[i], eng, scr, st, scr_elems)
                         : prox_fibers<T>(A, B, op, X, 0, g, L.scalar(i), nullptr, eng, scr, st, scr_elems);
    if (e == cudaSuccess && tp) e = nd_tape_pass<T>(tp, nt, p, X, g, L.scalar(i), st, lamf, fpi);
    return e;
}

const char* nd_terms(const int* ns, int nds, int npen, const double* dims, NdTerms* t) {
    long long n = 1;
    for (int i = 0; i < nds; i++) n *= ns[i];
    t->n = n;
    if (npen > 64) return "more than 64 penalty terms are not supported";
    for (int i = 0; i < npen; i++) {
        const int d = (int)(dims[i] - 1);                                     // TV2Dopt.cpp:171, TVNDopt.cpp:175
        if (d < 0 || d >= nds) return "invalid penalty dimensions";
        long long inc = 1;
        for (int a = 0; a < d; a++) inc *= ns[a];                             // TVNDopt.cpp:133-138
        t->g[i] = FiberGeom{ns[d] ? n / ns[d] : 0, ns[d], inc};
    }
    return nullptr;
}

static int read_stop(const double* dres, double* stop, cudaStream_t st) {
    cudaError_t e = cudaMemcpyAsync(stop, dres, sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e == cudaSuccess;
}

// The iteration of pd2_device and pd_device, over the running items of NdItems.  batch = 0 (the single-item entry points): one item that
// iterates in x_out with the single-item workspace (ws_bytes_pd(n, npen)), info nullptr allowed.  batch >= 1: a batch iterates in the
// workspace, and an item's x goes out when it stops.
// PD2_TV.  tape != nullptr (the recorded forward, dr2_vjp.cu): after each pass the segmentation tape of its output is written -- z as
// pass 2 iters, x as pass 2 iters + 1 (npen = 1: z as pass 0); nothing else changes.
template <typename T>
int pd2_device(const T* y, const double* lambdas, const double* dims, T* x_out, double* info, const int* ns, int nds, int npen,
               int maxIters, void* ws, Engine eng, cudaStream_t st, void* tape, int batch, int lstride) {
    if (npen > 2) { printf("PD2_TV: this algorithm can not work with more than 2 penalties\n");      // :95-96
                    if (info) info[INFO_RC] = RC_ERROR; return 0; }
    NdTerms t;
    const char* why = nd_terms(ns, nds, npen, dims, &t);
    const long long n = t.n;
    const int nb = batch > 0 ? batch : 1;
    if (maxIters <= 0) maxIters = MAX_ITERS_PD;
    NdPens<T> L(lambdas, lstride, npen >= 1 && npen <= 2 ? npen : 0, nb);
    if (npen >= 1 && npen <= 2) eng = lane_guard<T>(eng, y, n * nb, L.max(), st);
    if (npen < 1 || why) { printf("PD2_TV: invalid penalty dimensions\n"); if (info) info[INFO_RC] = RC_ERROR; return 0; }
    double row1[3];
    if (!info) info = row1;
    NdItems<T> I(nb, n, x_out, info);
    int iters = 0;
    if (n > 0) {
        const long long nt = n * nb;
        char* w = (char*)ws; const size_t ab = align256((size_t)nt * sizeof(T));
        T* p = (T*)w; w += ab; T* q = (T*)w; w += ab; T* z = (T*)w; w += ab; T* xl = (T*)w; w += ab;
        T* scr = (T*)w; w += 3 * ab;                 // staging of strided passes: 2 arrays + per-chunk masks / entering values
        double* scratch = (double*)w;
        I.split(batch ? (char*)ws + ws_bytes_pd<T>(nt, npen) : nullptr, scratch, scratch + REDUCE_BLOCKS);
        T* x = I.x;
        char* tp = tape ? (char*)tape + nd_tape_head_bytes(batch) : nullptr;
        T* const state[3] = {x, p, q};
        PTV_TRY(cudaMemcpyAsync(x, y, (size_t)nt * sizeof(T), cudaMemcpyDeviceToDevice, st));         // :132-137
        PTV_TRY(cudaMemsetAsync(p, 0, (size_t)nt * sizeof(T), st));
        PTV_TRY(cudaMemsetAsync(q, 0, (size_t)nt * sizeof(T), st));
        while (I.m > 0) {                                                                             // :157 per item
            const int m = I.m;
            const long long nm = n * m;
            const FiberGeom g0 = items_geom(t.g[0], m), g1 = npen >= 2 ? items_geom(t.g[1], m) : g0;
            PTV_TRY(L.sync(I, st));
            PTV_TRY(cudaMemcpyAsync(xl, x, (size_t)nm * sizeof(T), cudaMemcpyDeviceToDevice, st));
            PTV_TRY(nd_pass<T>(x, p, IN_A_PLUS_B, z, g0, t.g[0].nf, L, I, 0, eng, scr, 3 * nm, tp, nt, 2LL * iters, st));   // :171-208
            PTV_TRY(ew_dual_update<T>(p, x, z, nm, st));                                              // :211-213
            if (npen >= 2) {
                PTV_TRY(nd_pass<T>(z, q, IN_A_PLUS_B, x, g1, t.g[1].nf, L, I, 1, eng, scr, 3 * nm, tp, nt, 2LL * iters + 1, st));  // :216-258
                PTV_TRY(ew_dual_update<T>(q, z, x, nm, st));                                          // :261-263
            } else {
                PTV_TRY(cudaMemcpyAsync(x, z, (size_t)nm * sizeof(T), cudaMemcpyDeviceToDevice, st)); // :266-269
            }
            PTV_TRY(ew_mean_abs_diff_items<T>(x, xl, n, m, I.partial, I.dstop, st));                 // :273-277 per item
            iters++;
            // the loop condition (:157), one iteration only with one term; info rows (:283-295)
            PTV_TRY(I.step(iters, [&](double s) { return s > STOP_PD && npen > 1 && iters < maxIters; }, state, npen >= 2 ? 3 : 2,
                           scr, st));
        }
    }
    I.rest(0);
    return 1;
}

// The checks PD_TV and PDR_TV share, in this order: the term count; the lane guard over the largest penalty; the axes.  Refused:
// "<name>: <reason>" on stdout, info[RC] = RC_ERROR, false.
template <typename T>
static bool pd_start(const char* name, const T* y, const double* lam, const double* dims, double* info, const int* ns, int nds, int npen,
                     NdTerms* t, Engine* eng, cudaStream_t st, int items = 1, int lstride = 0) {
    const char* why = nd_terms(ns, nds, npen, dims, t);
    if (npen <= 64) {
        double lmax = 0.0;
        for (int b = 0; b < (lstride ? items : 1); b++) for (int i = 0; i < npen; i++) if (lam[(size_t)b * lstride + i] > lmax) lmax = lam[(size_t)b * lstride + i];
        *eng = lane_guard<T>(*eng, y, t->n * items, lmax, st);
    }
    if (why) { printf("%s: %s\n", name, why); if (info) info[INFO_RC] = RC_ERROR; return false; }
    return true;
}

// The workspace of pd_device and pdr_device (ws_bytes_pd): p_i and z_i of each term interleaved, the staging of strided passes (2
// arrays + per-chunk masks / entering values), the reduction scratch, then the device tables dp / dz of the p_i / z_i.
template <typename T> struct PdWs {
    T* hp[64]; T* hz[64];
    T* scr; double* scratch; double* dres;
    T** dp; T** dz;
};
template <typename T> static cudaError_t pd_ws(void* ws, long long n, int npen, PdWs<T>* W, cudaStream_t st) {
    char* w = (char*)ws; const size_t ab = align256((size_t)n * sizeof(T));
    for (int i = 0; i < npen; i++) { W->hp[i] = (T*)w; w += ab; W->hz[i] = (T*)w; w += ab; }
    W->scr = (T*)w; w += 3 * ab;
    W->scratch = (double*)w; W->dres = W->scratch + REDUCE_BLOCKS; w += SCRATCH_BYTES;
    W->dp = (T**)w; W->dz = W->dp + 64;
    cudaError_t e = cudaMemcpyAsync(W->dp, W->hp, sizeof(T*) * npen, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(W->dz, W->hz, sizeof(T*) * npen, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);    // W lives on the host stack
    return e;
}

// PD_TV, with pd2_device's items and workspaces.  tape != nullptr (the recorded forward, dr2_vjp.cu): after each pass the segmentation
// tape of its output p_i is written as pass iters * npen + i; nothing else changes.
template <typename T>
int pd_device(const T* y, const double* lam, const double* dims, T* x_out, double* info, const int* ns, int nds, int npen,
              int maxIters, void* ws, Engine eng, cudaStream_t st, void* tape, int batch, int lstride) {
    if (maxIters <= 0) maxIters = MAX_ITERS_PD;
    const int nb = batch > 0 ? batch : 1;
    NdTerms t;
    if (!pd_start<T>("PD_TV", y, lam, dims, info, ns, nds, npen, &t, &eng, st, nb, lstride)) return 0;
    const long long n = t.n, nt = n * nb;
    double row1[3];
    if (!info) info = row1;
    NdItems<T> I(nb, n, x_out, info);
    int iters = 0;
    if (n > 0 && npen > 0) {
        PdWs<T> W;
        PTV_TRY(pd_ws<T>(ws, nt, npen, &W, st));
        I.split(batch ? (char*)ws + ws_bytes_pd<T>(nt, npen) : nullptr, W.scratch, W.dres);
        T* x = I.x;
        char* tp = tape ? (char*)tape + nd_tape_head_bytes(batch) : nullptr;
        T* state[65] = {x};
        for (int i = 0; i < npen; i++) state[1 + i] = W.hz[i];
        PTV_TRY(cudaMemsetAsync(x, 0, (size_t)nt * sizeof(T), st));                                   // :125-130
        for (int i = 0; i < npen; i++) PTV_TRY(cudaMemcpyAsync(W.hz[i], y, (size_t)nt * sizeof(T), cudaMemcpyDeviceToDevice, st));
        NdPens<T> L(lam, lstride, npen, nb);
        while (I.m > 0) {                                                                             // :151 per item
            const int m = I.m;
            PTV_TRY(L.sync(I, st));
            for (int i = 0; i < npen; i++)                                                            // :171-208
                PTV_TRY(nd_pass<T>(W.hz[i], nullptr, IN_A, W.hp[i], items_geom(t.g[i], m), t.g[i].nf, L, I, i, eng, W.scr, 3 * n * m, tp, nt,
                                   (long long)iters * npen + i, st));
            PTV_TRY(ew_pd_combine_items<T>(W.dp, W.dz, W.hp, W.hz, npen, x, n, m, I.partial, I.dstop, st));   // :212-227 per item
            iters++;
            // the loop condition; info rows (:233-245)
            PTV_TRY(I.step(iters, [&](double s) { return s > STOP_PD && iters < maxIters; }, state, 1 + npen, W.scr, st));
        }
    } else if (n > 0) {
        PTV_TRY(cudaMemsetAsync(x_out, 0, (size_t)nt * sizeof(T), st));
    }
    I.rest(0);
    return 1;
}

// ------------------------------------------------------------------------------------------------------------------
// PDR_TV (src/TVNDopt.cpp:280-500): parallel Douglas-Rachford over k one-dimensional TV terms.  x = y / k, z_i = y; a FIXED
// number of iterations (the reference's loop has no stop test, :394) of  p_i = prox_{d_i}(z_i, k lam_i)  (1D solver: the
// reference calls TV1D_denoise, :439 -- the same minimiser as every other exact 1D solver here) ; q = mean p_i ; x = mean z_i ;
// z_i += 2 q - x - p_i ; stop = mean|x - x_last|.  The result x is the average of the z_i BEFORE the last update, like the
// reference's.  info = {iters, stop, RC_ITERS if iters >= 35 else RC_OK}; the stop value is read back once, after the loop.
// tape != nullptr (the recorded forward, dr2_vjp.cu): after each pass of the iterations but the last, the segmentation tape of its
// output p_i is written as pass j * npen + i of the tape; nothing else changes.
template <typename T>
int pdr_device(const T* y, const double* lam, const double* dims, T* x, double* info, const int* ns, int nds, int npen,
               int maxIters, void* ws, Engine eng, cudaStream_t st, void* tape) {
    if (maxIters <= 0) maxIters = MAX_ITERS_DR;                                                       // :320
    NdTerms t;
    if (!pd_start<T>("PDR_TV", y, lam, dims, info, ns, nds, npen, &t, &eng, st)) return 0;
    const long long n = t.n;
    double stop = 0; int iters = 0;
    if (n > 0 && npen > 0) {
        PdWs<T> W;
        PTV_TRY(pd_ws<T>(ws, n, npen, &W, st));
        PTV_TRY(ew_div_scalar<T>(y, x, n, (T)npen, st));                                              // :365-370
        for (int i = 0; i < npen; i++) PTV_TRY(cudaMemcpyAsync(W.hz[i], y, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));
        while (iters < maxIters) {                                                                    // :394
            for (int i = 0; i < npen; i++) {
                PTV_TRY(prox_fibers<T>(W.hz[i], nullptr, IN_A, W.hp[i], 0, t.g[i], (T)lam[i], nullptr, eng, W.scr, st, 3 * n));  // :409-449
                if (tape && iters < maxIters - 1)
                    PTV_TRY(pdr_tape_pass<T>(tape, n, (long long)iters * npen + i, W.hp[i], t.g[i], (T)lam[i], st));
            }
            PTV_TRY(ew_pdr_combine<T>(W.dp, W.dz, W.hp, W.hz, npen, x, n, W.scratch, W.dres, st));            // :456-475
            iters++;
        }
        if (iters > 0 && !read_stop(W.dres, &stop, st)) { PTV_TRY(cudaGetLastError()); PTV_TRY(cudaErrorUnknown); }
    } else if (n > 0) {
        PTV_TRY(cudaMemsetAsync(x, 0, (size_t)n * sizeof(T), st));
        iters = maxIters;
    }
    if (info) { info[INFO_ITERS] = iters; info[INFO_GAP] = stop;
                info[INFO_RC] = iters >= MAX_ITERS_DR ? RC_ITERS : RC_OK; }                           // :481-492
    return 1;
}

#define INST(T) \
    template size_t ws_bytes_dr2<T>(size_t, size_t, int); \
    template int dr2_device<T>(size_t, size_t, int, int, const T*, T, T, T*, int, double*, void*, Engine, cudaStream_t); \
    template int dr2_lane_pick<T>(size_t, size_t, int, int, const T*, const T*, const void*, T, T, Engine, void**); \
    template int drw_device<T>(size_t, size_t, int, int, const T*, const T*, const T*, T*, int, double*, void*, Engine, cudaStream_t); \
    template struct DrwPasses<T>; \
    template size_t ws_bytes_pd<T>(long long, int, int); \
    template int pd2_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t, \
                               void*, int, int); \
    template int pd_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t, \
                              void*, int, int); \
    template int pdr_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t, \
                               void*);
INST(double)
INST(float)

}  // namespace ptv
