// solver.cu -- device-resident outer loops: Douglas-Rachford (DR2_TV) and proximal Dykstra (PD2_TV, PD_TV).
//
// Semantics follow the reference exactly (same initialisation, pass order, iteration structure, stop test and info[]):
//   DR2_TV  src/TV2Dopt.cpp:352-444     PD2_TV  src/TV2Dopt.cpp:59-302     PD_TV  src/TVNDopt.cpp:48-252
// The reference's fixed 35 DR iterations are NOT a converged solve and the result depends on the pass order, so nothing
// here may be "improved" (SURVEY.md section 0.3).  All arrays stay in HBM for the whole solve; the only host round trip
// is the 8-byte stop criterion of the Dykstra loops, once per iteration.
#include "ptv_internal.h"
#include <float.h>
#include <stdio.h>

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
                                       const T* lamv, cudaStream_t st, T* X2 = nullptr, long long inc2 = 0);
template <typename T> cudaError_t gather_fibers_range(const T* A, const T* B, InOp op, T* out, FiberGeom g, int k_begin, int k_end, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_ex_range(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g,
                                    long long r_begin, long long r_end, cudaStream_t st);
template <typename T>
cudaError_t prox_fibers_chunked_contig_sparse(const T* A, T* X, FiberGeom g, T lam, const T* lamv, uint32_t* Mk, T* Cv, cudaStream_t st);
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
static constexpr int MAX_DEV = 64;
static DrPipe g_pipe_d[MAX_DEV];
static int cur_dev() { int d = 0; if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); d = 0; } return (d < 0 || d >= MAX_DEV) ? 0 : d; }
#define g_pipe (g_pipe_d[cur_dev()])

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
            if (sparse) PCHK(prox_fibers_chunked_contig_sparse<T>(t1 + r0 * (long long)N, t2 + r0 * (long long)N, FiberGeom{r1 - r0, (int)N, 1}, w2,
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
        if (!dr_iteration_pipelined<T>(g_pipe, M, N, Y, t, s, final ? out : x, scr, w1, w2, first, final, sparse, st)) {
            BTRY(cudaGetLastError()); return 1; }
        if (!final) { T* tmp = t; t = x; x = tmp; }
    }
    return 0;
#undef BTRY
}

// ------------------------------------------------------------------------------------------------------------------
// lane_guard (declared in ptv_internal.h): is the lane engine a good choice for this data?
struct LaneGuardState { const void* y = nullptr; long long n = 0; double lam = 0.0; size_t ts = 0; int ok = -1; double* dev = nullptr; };
static LaneGuardState g_guard_d[MAX_DEV];
int lane_guard_last() { return g_guard_d[cur_dev()].ok; }
template <typename T>
Engine lane_guard(Engine eng, const T* y, long long n, double lam, cudaStream_t st) {
    if (eng != ENGINE_AUTO || n < 2 || !(lam > 0.0)) return eng;
    LaneGuardState& G = g_guard_d[cur_dev()];
    {   // evaluated on every call: the same buffer (the C ABI's own staging area, a caller's frame buffer) holds different data each time
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) { cudaGetLastError(); return eng; }
        if (!G.dev && cudaMalloc(&G.dev, sizeof(double)) != cudaSuccess) { cudaGetLastError(); G.dev = nullptr; return ENGINE_CHUNKED; }
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
    const long long n = (long long)M * N * batch;
    LTRY(ew_image_means_x2<T>(Y, (long long)M * N, batch, t, scratch, st));                                   // t = 2 mean (:390-395)
    for (int it = 0; it <= maxit; it++) {
        const bool final = it == maxit, first = it == 0 && maxit > 0;
        if (first) LTRY(cudaMemcpyAsync(x1, t, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));
        else { KernelSpan sp(KC_PROX_CONTIG, 1, st);
               LTRY(ptvl::lane_prox<T>(ptvl::LANE_PLAIN, t, nullptr, nullptr, x1, (long long)N * batch, (int)M, 1, w1, lscr, st)); }
        { KernelSpan sp(KC_PROX_STRIDED, 1, st);
          LTRY(ptvl::lane_prox<T>(final ? ptvl::LANE_DR_B_FINAL : ptvl::LANE_DR_B, Y, x1, t, final ? out : t2, (long long)M * batch, (int)N,
                                  (long long)M, w2, lscr, st)); }
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
static DrGraph g_dr_graph_d[MAX_DEV];
#define g_dr_graph (g_dr_graph_d[cur_dev()])

// ------------------------------------------------------------------------------------------------------------------
template <typename T> size_t ws_bytes_dr2(size_t M, size_t N, int batch) {
    size_t n = M * N * (size_t)batch;
    return 7 * align256(n * sizeof(T)) + SCRATCH_BYTES;      // plain schedule: t, s, x, 2 staging; T-space schedule: 7 arrays
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
    const bool tspace = (eng == ENGINE_TSPACE || tpose) && !row_major && M >= 64 && N >= 64 && g_pipe.init();
    const bool piped = (eng == ENGINE_AUTO || eng == ENGINE_PIPELINED) && !row_major && batch == 1 && M >= 1024 && N >= 1024 && M % 2 == 0 && N % 2 == 0 &&
                       (size_t)((M > N ? M : N) * sizeof(T)) <= 96 * 1024 && g_pipe.init();
    // lane-per-fiber engine: images whose row pitch suits TMA tiling, positive weights.  Column-major: the staged schedule (column
    // pass over contiguous fibers) or, engine lane-t, the transposed one; row-major: only the transposed schedule applies.
    const void* lane_ptrs[3] = {Y, out, ws};
    void* lscr = nullptr;
    const bool lane_t = eng == ENGINE_LANE_T || row_major;
    bool lane = (eng == ENGINE_AUTO || eng == ENGINE_LANE || eng == ENGINE_LANE_T) && w1 > T(0) && w2 > T(0) && M >= 2 && N >= 2 && g_pipe.init() &&
                ptvl::lane_shape_ok((long long)N * batch, (int)M, lane_t ? (long long)N : 1, sizeof(T), lane_ptrs, 3) &&
                ptvl::lane_shape_ok((long long)M * batch, (int)N, (long long)M, sizeof(T), lane_ptrs, 3) &&
                (!lane_t || (((long long)M * sizeof(T)) % 16 == 0 && ((long long)N * sizeof(T)) % 16 == 0));
    if (lane) {
        void* a1 = ptvl::lane_scratch((long long)N * batch, (int)M); void* a2 = ptvl::lane_scratch((long long)M * batch, (int)N);
        lscr = a2; lane = a1 && a2;                 // the second call returns the (possibly grown) buffer both passes use
    }
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
            DrGraph& G = g_dr_graph;
            if (!(G.exec && G.key == key)) {
                if (G.exec) { cudaGraphExecDestroy(G.exec); G.exec = nullptr; }
                long long c0[KC_COUNT], c1[KC_COUNT];
                profile_counters(c0);
                cudaGraph_t graph = nullptr;
                bool okc = cudaStreamBeginCapture(g_pipe.sg, cudaStreamCaptureModeRelaxed) == cudaSuccess;
                if (okc) {
                    rc = body(g_pipe.sg);
                    okc = (cudaStreamEndCapture(g_pipe.sg, &graph) == cudaSuccess) && rc == 0 && graph;
                }
                if (okc) okc = cudaGraphInstantiate(&G.exec, graph, 0) == cudaSuccess;
                if (graph) cudaGraphDestroy(graph);
                profile_counters(c1);
                for (int i = 0; i < KC_COUNT; i++) { G.launches[i] = c1[i] - c0[i]; c1[i] = -G.launches[i]; }
                profile_add(c1);                                              // the capture itself launched nothing
                if (!okc) { cudaGetLastError(); G.exec = nullptr; } else G.key = key;
            }
            if (G.exec) {
                PTV_TRY(cudaEventRecord(g_pipe.eIn, st));
                PTV_TRY(cudaStreamWaitEvent(g_pipe.sg, g_pipe.eIn, 0));
                PTV_TRY(cudaGraphLaunch(G.exec, g_pipe.sg));
                PTV_TRY(cudaEventRecord(g_pipe.eOut, g_pipe.sg));
                PTV_TRY(cudaStreamWaitEvent(st, g_pipe.eOut, 0));
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
// DR2L1W_TV (src/TV2DWopt.cpp:46-140): the Douglas-Rachford skeleton of DR2_TV with per-edge weights -- W1: (M-1) x N
// (column fibers, contiguous, exactly the [fiber][len-1] layout of the weighted chunked kernel), W2: M x (N-1) (row
// fibers, stride M) -- and the opposite reflection signs (:115, :125).  Rows go through the same gather -> contiguous
// chunked kernel -> fused scatter route as DR2_TV; their weights are constant over the solve and are gathered once.
template <typename T> cudaError_t gather_fibers(const T* A, const T* B, InOp op, T* out, FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_ex(const T* in, const T* A, const T* B, const T* C, InOp op, int out_op, T* X, FiberGeom g, cudaStream_t st);
template <typename T>
cudaError_t scatter_fibers_sparse(const T* in, const uint32_t* Mk, const T* Cv, const T* A, const T* B, const T* C, InOp op, int out_op, T* X,
                                  FiberGeom g, cudaStream_t st);

template <typename T>
int drw_device(size_t M, size_t N, const T* Y, const T* W1, const T* W2, T* out, int maxit, double* info, void* ws, Engine eng,
               cudaStream_t st) {
    const long long n = (long long)M * (long long)N;
    if (maxit <= 0) maxit = MAX_ITERS_DR;                                     // TV2DWopt.cpp:82
    if (n == 0) { if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; } return 0; }
    char* w = (char*)ws;
    T* t = (T*)w; w += align256(n * sizeof(T));
    T* s = (T*)w; w += align256(n * sizeof(T));
    T* x = (T*)w; w += align256(n * sizeof(T));
    T* t1 = (T*)w; w += align256(n * sizeof(T));
    T* t2 = (T*)w; w += align256(n * sizeof(T));
    T* w2t = (T*)w; w += align256(n * sizeof(T));
    T* Cv = (T*)w; uint32_t* Mk = reinterpret_cast<uint32_t*>(Cv + (long long)M * (((long long)N + 31) / 32));   // sparse row results
    w += align256(n * sizeof(T));
    double* scratch = (double*)w;
    const FiberGeom gc{(long long)N, (int)M, 1}, gr{(long long)M, (int)N, (long long)M}, grc{(long long)M, (int)N, 1};
    bool fast_rows = eng != ENGINE_SEQ && N >= 64 && M >= 1;
    if (fast_rows) { KernelSpan sp(KC_ELEMENTWISE, 1, st);
                     PTV_TRY(gather_fibers<T>(W2, nullptr, IN_A, w2t, FiberGeom{(long long)M, (int)N - 1, (long long)M}, st)); }
    PTV_TRY(ew_image_means_x2<T>(Y, n, 1, t, scratch, st));                   // :85-89
    for (int it = 0; it <= maxit; it++) {                                     // :94-119, then the final pair :122-125
        const bool final = it == maxit;
        // columns: s = 2 (t - prox_W1(t)) - t   (final: s = t - prox_W1(t))
        PTV_TRY(prox_fibers_ex<T>(t, nullptr, nullptr, IN_A, s, final ? 2 : 1, gc, T(0), M > 1 ? W1 : nullptr, eng, nullptr, st, 0));
        // rows: in = Y - s ; tb = (in - prox_W2(in)) - Y ; tb = -2 tb - s ; t' = 0.5 (t + tb)   (final: out = -s - tb)
        T* dst = final ? out : x;
        const int oop = final ? 6 : 5;
        bool done = false;
        if (fast_rows) {
            { KernelSpan sp(KC_ELEMENTWISE, 1, st); PTV_TRY(gather_fibers<T>(Y, s, IN_A_MINUS_B, t1, gr, st)); }
            cudaError_t e;
            { KernelSpan sp(KC_PROX_STRIDED, 1, st);
              e = prox_fibers_chunked_contig_sparse<T>(t1, t2, grc, T(0), w2t, Mk, Cv, st);       // no fill: the scatter expands
              if (e == cudaErrorInvalidConfiguration) sp.cancel(); }
            if (e == cudaErrorInvalidConfiguration) { cudaGetLastError(); fast_rows = false; }
            else {
                PTV_TRY(e);
                KernelSpan sp(KC_ELEMENTWISE, 1, st);
                PTV_TRY(scatter_fibers_sparse<T>(t2, Mk, Cv, Y, s, t, IN_A_MINUS_B, oop, dst, gr, st));
                done = true;
            }
        }
        if (!done) PTV_TRY(prox_fibers_ex<T>(Y, s, t, IN_A_MINUS_B, dst, oop, gr, T(0), N > 1 ? W2 : nullptr, ENGINE_SEQ, nullptr, st, 0));
        if (!final) { T* tmp = t; t = x; x = tmp; }
    }
    if (info) { info[INFO_ITERS] = maxit; info[INFO_RC] = RC_OK; }            // :128-131
    return 0;                                                                 // :135 (returns 0 on success, like DR2_TV)
}

// ------------------------------------------------------------------------------------------------------------------
template <typename T> size_t ws_bytes_pd(long long n, int npen) {
    int arrays = 2 * npen + 4;   // PD_TV: p_i, z_i + 3 staging ; PD2_TV (npen <= 2): p, q, z, xl + 3 staging
    if (arrays < 8) arrays = 8;
    return (size_t)arrays * align256((size_t)n * sizeof(T)) + SCRATCH_BYTES + align256(2 * 64 * sizeof(void*));
}

static bool geom_of(const int* ns, int nds, double dim, long long n, FiberGeom* g) {
    int d = (int)(dim - 1);                                                   // TV2Dopt.cpp:171, TVNDopt.cpp:175
    if (d < 0 || d >= nds) return false;
    long long inc = 1;
    for (int i = 0; i < d; i++) inc *= ns[i];                                 // TVNDopt.cpp:133-138
    g->len = ns[d]; g->inc = inc; g->nf = ns[d] ? n / ns[d] : 0;
    return true;
}

static int read_stop(const double* dres, double* stop, cudaStream_t st) {
    cudaError_t e = cudaMemcpyAsync(stop, dres, sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e == cudaSuccess;
}

template <typename T>
int pd2_device(const T* y, const double* lambdas, const double* dims, T* x, double* info, const int* ns, int nds, int npen,
               int maxIters, void* ws, Engine eng, cudaStream_t st) {
    if (npen > 2) { printf("PD2_TV: this algorithm can not work with more than 2 penalties\n");      // :95-96
                    if (info) info[INFO_RC] = RC_ERROR; return 0; }
    long long n = 1; for (int i = 0; i < nds; i++) n *= ns[i];
    if (maxIters <= 0) maxIters = MAX_ITERS_PD;
    if (npen >= 1) eng = lane_guard<T>(eng, y, n, npen >= 2 && lambdas[1] > lambdas[0] ? lambdas[1] : lambdas[0], st);
    FiberGeom g0{0, 0, 1}, g1{0, 0, 1};
    if (npen < 1 || !geom_of(ns, nds, dims[0], n, &g0) || (npen >= 2 && !geom_of(ns, nds, dims[1], n, &g1))) {
        printf("PD2_TV: invalid penalty dimensions\n"); if (info) info[INFO_RC] = RC_ERROR; return 0; }
    double stop = DBL_MAX; int iters = 0;
    if (n > 0) {
        char* w = (char*)ws; const size_t ab = align256((size_t)n * sizeof(T));
        T* p = (T*)w; w += ab; T* q = (T*)w; w += ab; T* z = (T*)w; w += ab; T* xl = (T*)w; w += ab;
        T* scr = (T*)w; w += 3 * ab;                 // staging of strided passes: 2 arrays + per-chunk masks / entering values
        double* scratch = (double*)w; double* dres = scratch + REDUCE_BLOCKS;
        PTV_TRY(cudaMemcpyAsync(x, y, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));          // :132-137
        PTV_TRY(cudaMemsetAsync(p, 0, (size_t)n * sizeof(T), st));
        PTV_TRY(cudaMemsetAsync(q, 0, (size_t)n * sizeof(T), st));
        while (stop > STOP_PD && (npen > 1 || !iters) && iters < maxIters) {                           // :157
            PTV_TRY(cudaMemcpyAsync(xl, x, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));
            PTV_TRY(prox_fibers<T>(x, p, IN_A_PLUS_B, z, 0, g0, (T)lambdas[0], nullptr, eng, scr, st, 3 * n));       // :171-208
            PTV_TRY(ew_dual_update<T>(p, x, z, n, st));                                               // :211-213
            if (npen >= 2) {
                PTV_TRY(prox_fibers<T>(z, q, IN_A_PLUS_B, x, 0, g1, (T)lambdas[1], nullptr, eng, scr, st, 3 * n));   // :216-258
                PTV_TRY(ew_dual_update<T>(q, z, x, n, st));                                           // :261-263
            } else {
                PTV_TRY(cudaMemcpyAsync(x, z, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));  // :266-269
            }
            PTV_TRY(ew_mean_abs_diff<T>(x, xl, n, scratch, dres, st));                                // :273-277
            if (!read_stop(dres, &stop, st)) { PTV_TRY(cudaGetLastError()); PTV_TRY(cudaErrorUnknown); }
            iters++;
        }
    }
    if (info) { info[INFO_ITERS] = iters; info[INFO_GAP] = stop;
                info[INFO_RC] = iters >= MAX_ITERS_PD ? RC_ITERS : RC_OK; }                           // :283-295
    return 1;
}

template <typename T>
int pd_device(const T* y, const double* lam, const double* dims, T* x, double* info, const int* ns, int nds, int npen,
              int maxIters, void* ws, Engine eng, cudaStream_t st) {
    long long n = 1; for (int i = 0; i < nds; i++) n *= ns[i];
    if (maxIters <= 0) maxIters = MAX_ITERS_PD;
    if (npen > 64) { printf("PD_TV: more than 64 penalty terms are not supported\n"); if (info) info[INFO_RC] = RC_ERROR; return 0; }
    { double lmax = 0.0; for (int i = 0; i < npen; i++) if (lam[i] > lmax) lmax = lam[i];
      eng = lane_guard<T>(eng, y, n, lmax, st); }
    FiberGeom g[64];
    for (int i = 0; i < npen; i++)
        if (!geom_of(ns, nds, dims[i], n, &g[i])) { printf("PD_TV: invalid penalty dimensions\n");
                                                     if (info) info[INFO_RC] = RC_ERROR; return 0; }
    double stop = DBL_MAX; int iters = 0;
    if (n > 0 && npen > 0) {
        char* w = (char*)ws; const size_t ab = align256((size_t)n * sizeof(T));
        T* hp[64]; T* hz[64];
        for (int i = 0; i < npen; i++) { hp[i] = (T*)w; w += ab; hz[i] = (T*)w; w += ab; }
        T* scr = (T*)w; w += 3 * ab;
        double* scratch = (double*)w; double* dres = scratch + REDUCE_BLOCKS; w += SCRATCH_BYTES;
        T** dp = (T**)w; T** dz = dp + 64;
        PTV_TRY(cudaMemcpyAsync(dp, hp, sizeof(T*) * npen, cudaMemcpyHostToDevice, st));
        PTV_TRY(cudaMemcpyAsync(dz, hz, sizeof(T*) * npen, cudaMemcpyHostToDevice, st));
        PTV_TRY(cudaStreamSynchronize(st));    // hp/hz are stack arrays
        PTV_TRY(cudaMemsetAsync(x, 0, (size_t)n * sizeof(T), st));                                    // :125-130
        for (int i = 0; i < npen; i++) PTV_TRY(cudaMemcpyAsync(hz[i], y, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));
        while (stop > STOP_PD && iters < maxIters) {                                                  // :151
            for (int i = 0; i < npen; i++)
                PTV_TRY(prox_fibers<T>(hz[i], nullptr, IN_A, hp[i], 0, g[i], (T)lam[i], nullptr, eng, scr, st, 3 * n));  // :171-208
            PTV_TRY(ew_pd_combine<T>(dp, dz, hp, hz, npen, x, n, scratch, dres, st));                         // :212-227
            if (!read_stop(dres, &stop, st)) { PTV_TRY(cudaGetLastError()); PTV_TRY(cudaErrorUnknown); }
            iters++;
        }
    } else if (n > 0) {
        PTV_TRY(cudaMemsetAsync(x, 0, (size_t)n * sizeof(T), st));
    }
    if (info) { info[INFO_ITERS] = iters; info[INFO_GAP] = stop;
                info[INFO_RC] = iters >= MAX_ITERS_PD ? RC_ITERS : RC_OK; }                           // :233-245
    return 1;
}

// ------------------------------------------------------------------------------------------------------------------
// PDR_TV (src/TVNDopt.cpp:280-500): parallel Douglas-Rachford over k one-dimensional TV terms.  x = y / k, z_i = y; a FIXED
// number of iterations (the reference's loop has no stop test, :394) of  p_i = prox_{d_i}(z_i, k lam_i)  (1D solver: the
// reference calls TV1D_denoise, :439 -- the same minimiser as every other exact 1D solver here) ; q = mean p_i ; x = mean z_i ;
// z_i += 2 q - x - p_i ; stop = mean|x - x_last|.  The result x is the average of the z_i BEFORE the last update, like the
// reference's.  info = {iters, stop, RC_ITERS if iters >= 35 else RC_OK}; the stop value is read back once, after the loop.
template <typename T>
int pdr_device(const T* y, const double* lam, const double* dims, T* x, double* info, const int* ns, int nds, int npen,
               int maxIters, void* ws, Engine eng, cudaStream_t st) {
    long long n = 1; for (int i = 0; i < nds; i++) n *= ns[i];
    if (maxIters <= 0) maxIters = MAX_ITERS_DR;                                                       // :320
    if (npen > 64) { printf("PDR_TV: more than 64 penalty terms are not supported\n"); if (info) info[INFO_RC] = RC_ERROR; return 0; }
    { double lmax = 0.0; for (int i = 0; i < npen; i++) if (lam[i] > lmax) lmax = lam[i];
      eng = lane_guard<T>(eng, y, n, lmax, st); }
    FiberGeom g[64];
    for (int i = 0; i < npen; i++)
        if (!geom_of(ns, nds, dims[i], n, &g[i])) { printf("PDR_TV: invalid penalty dimensions\n");
                                                     if (info) info[INFO_RC] = RC_ERROR; return 0; }
    double stop = 0; int iters = 0;
    if (n > 0 && npen > 0) {
        char* w = (char*)ws; const size_t ab = align256((size_t)n * sizeof(T));
        T* hp[64]; T* hz[64];
        for (int i = 0; i < npen; i++) { hp[i] = (T*)w; w += ab; hz[i] = (T*)w; w += ab; }
        T* scr = (T*)w; w += 3 * ab;
        double* scratch = (double*)w; double* dres = scratch + REDUCE_BLOCKS; w += SCRATCH_BYTES;
        T** dp = (T**)w; T** dz = dp + 64;
        PTV_TRY(cudaMemcpyAsync(dp, hp, sizeof(T*) * npen, cudaMemcpyHostToDevice, st));
        PTV_TRY(cudaMemcpyAsync(dz, hz, sizeof(T*) * npen, cudaMemcpyHostToDevice, st));
        PTV_TRY(cudaStreamSynchronize(st));    // hp/hz are stack arrays
        PTV_TRY(ew_div_scalar<T>(y, x, n, (T)npen, st));                                              // :365-370
        for (int i = 0; i < npen; i++) PTV_TRY(cudaMemcpyAsync(hz[i], y, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, st));
        while (iters < maxIters) {                                                                    // :394
            for (int i = 0; i < npen; i++)
                PTV_TRY(prox_fibers<T>(hz[i], nullptr, IN_A, hp[i], 0, g[i], (T)lam[i], nullptr, eng, scr, st, 3 * n));  // :409-449
            PTV_TRY(ew_pdr_combine<T>(dp, dz, hp, hz, npen, x, n, scratch, dres, st));                        // :456-475
            iters++;
        }
        if (iters > 0 && !read_stop(dres, &stop, st)) { PTV_TRY(cudaGetLastError()); PTV_TRY(cudaErrorUnknown); }
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
    template int drw_device<T>(size_t, size_t, const T*, const T*, const T*, T*, int, double*, void*, Engine, cudaStream_t); \
    template size_t ws_bytes_pd<T>(long long, int); \
    template int pd2_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t); \
    template int pd_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t); \
    template int pdr_device<T>(const T*, const double*, const double*, T*, double*, const int*, int, int, int, void*, Engine, cudaStream_t);
INST(double)
INST(float)

}  // namespace ptv
