// ptv_internal.h -- internal host-side declarations shared by the CUDA translation units of libproxtv_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace ptv {

// Return codes and info slots of the reference (src/general.h:58-73).
enum { INFO_ITERS = 0, INFO_GAP = 1, INFO_RC = 2 };
enum { RC_OK = 0, RC_ITERS = 1, RC_STUCK = 2, RC_ERROR = 3 };
constexpr double STOP_PD = 1e-6;       // src/TVopt.h:71
constexpr int MAX_ITERS_PD = 35;       // src/TVopt.h:73
constexpr int MAX_ITERS_DR = 35;       // src/TVopt.h:83

// State kept per device (workspaces, streams, graphs, scratch) lives in tables of MAX_DEVICES slots, indexed by device_slot(): the
// current device's index, or -1 when there is none or it lies past the table (the caller then refuses, or answers "none").
constexpr int MAX_DEVICES = 64;
inline int device_slot() {
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); return -1; }
    return d >= 0 && d < MAX_DEVICES ? d : -1;
}

// The set of 1D fibers of a column-major array along one dimension (src/TVNDopt.cpp:133-138,184-188):
// fiber j starts at (j / inc) * inc * len + (j % inc) and its elements are `inc` apart.  A leading batch of arrays is
// simply one more (slowest) dimension.
struct FiberGeom {
    long long nf;    // number of fibers
    int len;         // samples per fiber
    long long inc;   // element stride inside a fiber (1 = contiguous fibers)
};

// How a fiber's input is formed from up to two arrays, and what is written back (fused DR / Dykstra arithmetic).
enum InOp { IN_A = 0, IN_A_MINUS_B = 1, IN_A_PLUS_B = 2 };

// Which kernel family prox_fibers() may use.
enum Engine { ENGINE_AUTO = 0, ENGINE_SEQ = 1, ENGINE_CHUNKED = 2, ENGINE_CHUNKED_STRIDED = 3, ENGINE_PIPELINED = 4, ENGINE_TSPACE = 5, ENGINE_TPOSE = 6,
              ENGINE_LANE = 7 /* lane-per-fiber streaming engine (kernels_lane.cu); what AUTO uses when the shape suits TMA tiling */,
              ENGINE_LANE_T = 8 /* DR2_TV only: lane engine, both passes strided with transposed results (dr2_lane_t_body) */ };

struct ProxStats {           // filled asynchronously on the device; optional
    unsigned long long fallback_fibers;
};

// x = prox_{lam * TV}(in) for every fiber.  lamv == nullptr: uniform weight lam; else per-edge weights, laid out like the
// fibers but with len-1 samples per fiber.  All pointers are device pointers.  Returns cudaGetLastError().
// out_op (OutOp in chunk_core.cuh): 0 X = prox ; 1 X = 2*(in - prox) - in (DR reflection) ; 2 X = in - prox.
template <typename T>
cudaError_t prox_fibers(const T* A, const T* B, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv, Engine eng,
                        T* scratch /* 2 * nf * len elements, or nullptr */, cudaStream_t st,
                        long long scratch_elems = 0 /* actual size if larger than the 2n convention (long contiguous fibers) */);

// Same, with a third array C for the fused Douglas-Rachford row pass (out_op 3 / 4, see OutOp in chunk_core.cuh).
template <typename T>
cudaError_t prox_fibers_ex(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, const T* lamv,
                           Engine eng, T* scratch, cudaStream_t st, long long scratch_elems = 0, const T* lamf = nullptr, long long fpi = 1,
                           bool lamf_pos = false);
// prox_fibers with out_op 0, no per-edge weights and one penalty per group of fpi fibers: fiber j's is lamf[j / fpi] (device table,
// fpi >= 1), and its result equals bit for bit the uniform pass with that penalty on the kernel family that ran it (the routes that
// decline a table: prox_dispatch.cu).  pos: every entry of the table is > 0 (the lane engine takes only such tables).
template <typename T>
cudaError_t prox_fibers_lamf(const T* A, const T* B, InOp op, T* X, FiberGeom g, const T* lamf, long long fpi, bool pos, Engine eng, T* scratch,
                             cudaStream_t st, long long scratch_elems = 0);

long long strided_scratch_elems(long long nf, long long len);   // scratch elements that enable the sparse strided route (else 2n: dense route)
long long lf_scratch_elems(long long nf, long long len);     // scratch elements prox_fibers needs for contiguous fibers longer than shared memory
// tests: what the long-fiber tiles (long_fiber.cu) did in the latest batched 1D prox entry call on this device -- 1 used, 0 tried and
// fell back to the sequential kernel, -1 not tried.  The entry points note -1 before they dispatch; prox_fibers_ex notes 1 or 0.
void long_fiber_note(int v);
int long_fiber_last();

// ---- launch accounting / event timing (profile.cu) ----
enum KernelClass { KC_PROX_CONTIG = 0, KC_PROX_STRIDED = 1, KC_ELEMENTWISE = 2, KC_COUNT = 3 };
struct KernelSpan {          // RAII: counts `nkernels` launches of class cls; when profiling is on, brackets them with events
    int cls; cudaStream_t st; cudaEvent_t a;
    KernelSpan(int cls, int nkernels, cudaStream_t st);
    ~KernelSpan();
    void cancel();      // the bracketed launch did not happen: undo the count, drop the timing
};
void profile_enable(int on);
void profile_reset();
void profile_read(double* ms, long long* launches, long long* spans);   // arrays of KC_COUNT
bool profile_is_enabled();
void profile_counters(long long* out);          // current launch counters (KC_COUNT)
void profile_add(const long long* delta);       // account for a CUDA-graph replay

// ---- elementwise helpers (elementwise.cu) ----
template <typename T> cudaError_t ew_image_means_x2(const T* Y, long long per_image, int batch, T* t, double* scratch,
                                                    cudaStream_t st);                 // t[b,:] = 2*mean(Y[b,:])
template <typename T> cudaError_t ew_dr_reflect_cols(const T* t, const T* x, T* s, long long n, cudaStream_t st);
template <typename T> cudaError_t ew_dr_combine_rows(const T* Y, const T* s, const T* x, T* t, long long n, cudaStream_t st);
template <typename T> cudaError_t ew_dr_final_cols(const T* t, const T* x, T* s, long long n, cudaStream_t st);
template <typename T> cudaError_t ew_dr_final_rows(const T* Y, const T* s, const T* x, T* out, long long n, cudaStream_t st);
template <typename T> cudaError_t ew_dr_reflect_bcast(const T* t, const T* x1, T* s, long long n, long long per_image, int len,
                                                      long long inc, cudaStream_t st);
template <typename T> cudaError_t prox_const_fibers(const T* c, long long c_stride, int batch, int n, T lam, T* x1, cudaStream_t st);
template <typename T> cudaError_t ew_dual_update(T* p, const T* a, const T* b, long long n, cudaStream_t st);  // p += a - b
template <typename T> cudaError_t ew_pdr_combine(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                 double* scratch, double* result, cudaStream_t st);
template <typename T> cudaError_t ew_div_scalar(const T* y, T* x, long long n, T k, cudaStream_t st);             // x = y / k
template <typename T> cudaError_t ew_mean_abs_step(const T* y, long long n, double* out, cudaStream_t st);       // out[0] = mean |y[e+1] - y[e]|; out[1..256]: scratch
template <typename T> cudaError_t ew_dr_first(const T* Y, const T* t, T* U, T* D, long long n, cudaStream_t st);  // D = t - t ; U = Y - (2 D - t)
constexpr int REDUCE_BLOCKS = 1184;    // fixed, not the device's SM count (~9 per SM on a 132-SM H100): partial sums are combined in
                                       // the same fixed order on every GPU (deterministic)
// PD_TV's combine and PD2_TV's mean|a - b| with a stop value per item (DESIGN.md section 16): `items` running items of n elements in
// slots 0..items-1 of each array (a single-item solve: one item); result[s] = slot s's stop value, the same bits whichever slot the
// item sits in.  scratch: items * REDUCE_BLOCKS doubles.
template <typename T> cudaError_t ew_pd_combine_items(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                      int items, double* scratch, double* result, cudaStream_t st);
template <typename T> cudaError_t ew_mean_abs_diff_items(const T* a, const T* b, long long n, int items, double* scratch, double* result,
                                                         cudaStream_t st);
// dst slot s (n elements) = src slot map[s] (device array), or for map[s] = -1 - b item b's start value (init 0: 0, 1: G_b / kk,
// 2: G_b / kk - 0, 3: G_b - 0); src and dst must not overlap
template <typename T> cudaError_t ew_slot_gather(const T* src, T* dst, const int* map, int slots, long long n, int init, const T* G, T kk,
                                                 cudaStream_t st);

// ---- device-resident solvers (solver.cu).  All arrays are device pointers; `ws` must hold ws_bytes_*() bytes. ----
template <typename T> size_t ws_bytes_dr2(size_t M, size_t N, int batch);
template <typename T> int dr2_device(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit, double* info,
                                     void* ws, Engine eng, cudaStream_t st);
// DR2L1W_TV on `batch` M x N images back to back, column-major (row_major = 0) or C order (1); W1: (M-1) x N, W2: M x (N-1) per image,
// back to back, each laid out by the fiber rule of its pass (len - 1 samples per fiber); workspace of ws_bytes_dr2(M, N, batch) bytes
template <typename T> int drw_device(size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit,
                                     double* info, void* ws, Engine eng, cudaStream_t st);
// The prox passes of the weighted solve, shared by drw_device and drw_record_device (solver.cu).  axis 0: the column pass (fibers of
// length M, weights W1), axis 1: the row pass (length N, W2).  The strided axis of the storage order: gather (input op fused) ->
// contiguous weighted chunked kernel with a sparse result -> scatter (output form fused while it expands); the other: the chunked kernel with its fill, or
// for the weighted Douglas-Rachford forms the sparse result and expand_fibers_sparse (transpose.cu).  ENGINE_SEQ, fibers shorter than
// 64 and a refused chunked launch: the sequential kernel.  The strided pass's weights are gathered once, by init().
template <typename T> struct DrwPasses {
    FiberGeom g[2];
    const T* W[2];
    Engine eng;
    int strided;                 // the axis that takes the gather route: 1 (rows) for column-major images, 0 (columns) for C order
    bool fast[2];
    T *t1, *t2, *wg, *Cv; uint32_t* Mk;
    // stage: 4 arrays of M N batch elements (align256 each)
    cudaError_t init(size_t M, size_t N, int batch, int row_major, const T* W1, const T* W2, Engine eng, void* stage, cudaStream_t st);
    cudaError_t run(int axis, const T* A, const T* B, const T* C, InOp op, T* X, int out_op, cudaStream_t st);
};
// ---- the N-D solvers PD2_TV, PD_TV, PDR_TV (solver.cu; backward passes in dr2_vjp.cu) ----
enum NdSolver { ND_PD2 = 0, ND_PD = 1, ND_PDR = 2 };
// The element count of a column-major array of dims ns[0..nds) and the fibers of each penalty term along it
struct NdTerms {
    long long n;
    FiberGeom g[64];
};
// Fills t: n, then the fibers of term i along its 1-based axis dims[i] (npen = 0: n only).  nullptr when every axis is valid, else the
// reason: more than 64 terms (no fibers filled) or an axis outside 1..nds.
const char* nd_terms(const int* ns, int nds, int npen, const double* dims, NdTerms* t);
// the forward workspace of the three N-D solvers for n elements and npen terms; batch >= 1: of the batched PD_TV / PD2_TV solve
template <typename T> size_t ws_bytes_pd(long long n, int npen, int batch = 0);
// The slot rule of the batched PD_TV / PD2_TV (DESIGN.md section 16), the one place forward and backward take it from: at iteration j
// (0-based) the state arrays hold the items {b : K[b] > j}, in increasing b, in slots 0, 1, ...  Writes them to slots (unless nullptr)
// and returns their count.  The forward runs it with K[b] = INT_MAX for an item that has not stopped yet.
int nd_slots(const int* K, int batch, int j, int* slots);
// PD2_TV / PD_TV (proximal Dykstra, stop rule mean|x - x_old| <= STOP_PD).  tape: nullptr, or the recorded forward's buffer (header
// written by the caller after the call, from info[0]): the segmentation tape of every pass.
// batch = 0: one array (the single-item entry points).  batch >= 1: `batch` items of prod(ns) elements back to back in y and x, each
// with its own stop rule and info row (info: 3 batch doubles), bit for bit the single-item call on that item under the seq and chunked
// engines; tape: the batched layout (nd_tape_head_bytes(batch) bytes of header and K table, then passes of batch items each).
// lstride: the penalties' row stride -- 0, one row lambdas[0..npen) for every item; npen (batch >= 1), item b's row at lambdas + b npen
// (DESIGN.md section 16.1): item b is then solved with its own row, bit for bit as the single-item call with that row under the seq and
// chunked engines.
template <typename T> int pd2_device(const T* y, const double* lambdas, const double* dims, T* x, double* info, const int* ns,
                                     int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st, void* tape = nullptr,
                                     int batch = 0, int lstride = 0);
template <typename T> int pd_device(const T* y, const double* lambdas_scaled, const double* dims, T* x, double* info,
                                    const int* ns, int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st,
                                    void* tape = nullptr, int batch = 0, int lstride = 0);
// Engine choice under ENGINE_AUTO for data y (device pointer, n elements) and penalty lam: the lane engine keeps every open segment of
// a fiber inside a 64-row (float64) / 128-row (float32) shared-memory window and sends fibers whose segments outgrow it through a
// slow exact repair path, so it only pays while segments are short -- lam not larger than about the mean step |y[i+1] - y[i]| of the
// data (the repair count of a 4096 x 4096 solve explodes from 13 to 1.9 million between lam = 0.57 and 2.9 mean steps, and the
// repairs run one fiber at a time, so the solve becomes far slower than on the chunked engine).  Returns ENGINE_CHUNKED when eng is AUTO and the data does not suit the
// lane engine, else eng.  One small kernel and one stream synchronisation per call (the data behind a pointer changes between calls).
template <typename T> Engine lane_guard(Engine eng, const T* y, long long n, double lam, cudaStream_t st);
int lane_guard_last();           // tools / tests: last decision on this device (1 lane suits, 0 it does not, -1 none taken)
// The lane schedule dr2_device takes for these arguments and engine (already through lane_guard): 0 none, 1 staged (dr2_lane_body),
// 2 transposed (dr2_lane_t_body).  A lane schedule gets the lane engine's scratch in *lscr (allocates: call outside stream capture).
template <typename T> int dr2_lane_pick(size_t M, size_t N, int batch, int row_major, const T* Y, const T* out, const void* ws, T w1, T w2,
                                        Engine eng, void** lscr);

// ---- exact backward pass of DR2_TV (dr2_vjp.cu, DESIGN.md section 11) ----
size_t dr2_tape_bytes(size_t M, size_t N, int batch, int maxit);          // header + (2K + 1) passes x two bitsets
template <typename T> size_t ws_bytes_dr2_record(size_t M, size_t N, int batch);
template <typename T> size_t ws_bytes_dr2_vjp(size_t M, size_t N, int batch);
// DR2_TV with the schedule of the lane engine in plain passes, writing the segmentation tape of every pass but the first column pass.
// The tape's size (dr2_tape_bytes) is checked by the caller.  Returns a CUDA error (cudaErrorInvalidConfiguration: a lane pass refused).
template <typename T> cudaError_t dr2_record_device(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit,
                                                    void* tape, void* ws, Engine eng, cudaStream_t st);
// Validates a tape's header against the arguments (host; reads it back with one stream synchronisation): nullptr ok, else the reason.
const char* dr2_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, int maxit, cudaStream_t st);
template <typename T> cudaError_t dr2_vjp_device(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout,
                                                 T* gY, double* glam, void* ws, cudaStream_t st);
// ---- exact backward pass of DR2L1W_TV (dr2_vjp.cu, DESIGN.md section 12) ----
size_t drw_tape_bytes(size_t M, size_t N, int batch, int maxit);         // header + (2K + 2) passes x two bitsets
template <typename T> size_t ws_bytes_drw_record(size_t M, size_t N, int batch);
template <typename T> size_t ws_bytes_drw_vjp(size_t M, size_t N, int batch);
// drw_device's iteration with plain prox passes (bit for bit the same output), writing the segmentation tape of every pass.  The
// tape's size (drw_tape_bytes) and the arguments are checked by the caller.
template <typename T> cudaError_t drw_record_device(size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out,
                                                    int maxit, void* tape, void* ws, Engine eng, cudaStream_t st);
const char* drw_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, int maxit, cudaStream_t st);
// gY, and per-edge gW1 / gW2 unless nullptr, from the tape alone
template <typename T> cudaError_t drw_vjp_device(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout,
                                                 T* gY, T* gW1, T* gW2, void* ws, cudaStream_t st);

// PDR_TV (src/TVNDopt.cpp:280-500): parallel Douglas-Rachford, fixed iteration count; same workspace as pd_device.  tape: nullptr, or
// the recorded forward's buffer (header written by the caller): the segmentation tape of every pass but the last iteration's
template <typename T> int pdr_device(const T* y, const double* lambdas_scaled, const double* dims, T* x, double* info,
                                     const int* ns, int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st,
                                     void* tape = nullptr);
// ---- exact backward passes of the N-D solvers (dr2_vjp.cu, DESIGN.md sections 13 and 14) ----
// The tape of a recorded forward: a 256-byte header, then the segmentation tape of each pass that reaches the output.  maxIters <= 0
// means the solver's default (35).  PDR_TV runs K = maxIters iterations and records the (K - 1) npen passes of all but the last; PD_TV
// and PD2_TV stop early, so their tape holds the capacity of maxIters iterations -- maxIters npen passes (PD_TV), 2 maxIters (PD2_TV; 1
// when npen = 1) -- and the header the iterations run, `iters` (info[0]; ignored for PDR_TV).
constexpr int PDR_TAPE_MAX_DIMS = 16;                                    // axes the tape header holds
// header + passes x two bitsets; 0 when the byte count does not fit in size_t.  batch >= 1: the batched PD_TV / PD2_TV tape (section 16),
// whose passes hold `batch` items each
size_t nd_tape_bytes(NdSolver s, const int* ns, int nds, int npen, int maxIters, int batch = 0);
// the bytes before the first pass: the 256-byte header, and for batch >= 1 the K table (batch int32, 256-byte aligned)
size_t nd_tape_head_bytes(int batch);
// the tape of pass p (output y over the fibers g, penalty lam) into a tape of n-element passes
template <typename T> cudaError_t pdr_tape_pass(void* tape, long long n, long long p, const T* y, FiberGeom g, T lam, cudaStream_t st);
// the same into the passes that start at `passes`, each sized for cap_n elements (y covers the first nf * len of them)
// lamf != nullptr: fiber j's penalty is lamf[j / fpi] instead of lam (fiber_tape_lamf)
template <typename T> cudaError_t nd_tape_pass(void* passes, long long cap_n, long long p, const T* y, FiberGeom g, T lam, cudaStream_t st,
                                               const T* lamf = nullptr, long long fpi = 1);
// writes the 256-byte header after the solve (arguments checked by the caller; axes = dims - 1)
cudaError_t nd_tape_header(NdSolver s, void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters,
                           cudaStream_t st);
// validates a tape's header against the arguments (one stream synchronisation): nullptr ok, else the reason
const char* nd_tape_check(NdSolver s, const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                          int iters, cudaStream_t st);
// The batched tape's header and K table (K[b] = info[3 b]), written after the solve; and its check, which also reads the K table into K
// (batch ints) -- one stream synchronisation for both
cudaError_t nd_tape_header_batched(NdSolver s, void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                                   int batch, const double* info, cudaStream_t st);
const char* nd_tape_check_batched(NdSolver s, const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims,
                                  int maxIters, int batch, int* K, cudaStream_t st);
template <typename T> size_t ws_bytes_nd_vjp(const NdTerms& t, int npen, bool want_glam, int batch = 0);
// gY, and glam[npen] unless nullptr (PD_TV / PDR_TV: d/d of the scaled penalties; PD2_TV: of the penalties as given), from the tape
// alone; arguments checked by the caller; workspace ws_bytes_nd_vjp.  batch >= 1 (PD_TV / PD2_TV): the batched tape, item b's K = Kb[b]
// (host), glam[batch][npen] of the penalties as given for both solvers
template <typename T> cudaError_t nd_vjp_device(NdSolver s, const NdTerms& t, int npen, int maxIters, int iters, const void* tape,
                                                const T* gout, T* gY, double* glam, void* ws, cudaStream_t st, int batch = 0,
                                                const int* Kb = nullptr);

// ---- CondatChambollePock2_TV (cp2.cu, DESIGN.md section 15): Condat (alg 0), Chambolle-Pock (1) and accelerated Chambolle-Pock (2) ----
size_t ws_bytes_cp2(size_t M, size_t N, int batch, size_t elem);
// `batch` M x N images back to back, column-major (row_major = 0) or C order (1); alg in 0..2 (checked by the caller); maxit <= 0:
// 2500.  iters: nullptr, or host memory for each image's final `it` (iterations run + 1; the call then synchronises the stream).
// Reads the running-image count back every 64 iterations (one stream synchronisation each).  weighted (section 15.1; alg 0 or 1,
// lambda unused): each dual is clipped to its edge's weight in W1 ((M-1) x N per image) / W2 (M x (N-1)), device maps laid out like
// proxtv_DR2L1W_TV_batched_*'s; W1 may be nullptr when M == 1, W2 when N == 1.  The workspace is the same either way.  tape: nullptr, or
// a buffer of cp2_tape_bytes() bytes (alg 0 or 1, M N < 2^31; checked by the caller) that cp2_tape_tail fills after the solve.
template <typename T>
cudaError_t cp2_device(size_t M, size_t N, int batch, int row_major, const T* Y, double lambda, bool weighted, const T* W1, const T* W2,
                       T* out, int alg, int maxit, int* iters, void* ws, cudaStream_t st, void* tape = nullptr);
// ---- backward pass of the converged solve (cp2_vjp.cu, DESIGN.md section 15.2) ----
size_t cp2_tape_bytes(size_t M, size_t N, int batch);                   // 256-byte header + two bitsets (fused along F, along S)
size_t ws_bytes_cp2_vjp(size_t M, size_t N, int batch);
// The fused-edge tape of a finished solve: X its result, Uf / Us the two buffers of each dual, image b's final ones those of iteration
// (stopped[b] ? stopped[b] : it_end) - 1; Wf / Ws the weight maps in storage terms (weighted), else lambda.
template <typename T>
cudaError_t cp2_tape_tail(size_t M, size_t N, int batch, int row_major, const T* X, const T* const Uf[2], const T* const Us[2], const int* stopped,
                          int it_end, double lambda, bool weighted, const T* Wf, const T* Ws, void* tape, cudaStream_t st);
// Validates a tape's header against the arguments (one stream synchronisation): nullptr ok, else the reason.
const char* cp2_tape_check(const void* tape, size_t elem, size_t M, size_t N, int batch, int row_major, bool weighted, cudaStream_t st);
// gY (laid out like X), per-edge gW1 / gW2 (like W1 / W2) unless nullptr, glam[2 batch] unless nullptr, from the tape, the forward's
// result X and the upstream gradient gout; workspace ws_bytes_cp2_vjp().  Arguments checked by the caller.
template <typename T>
cudaError_t cp2_vjp_device(size_t M, size_t N, int batch, int row_major, const void* tape, const T* X, const T* gout, T* gY, T* gW1, T* gW2,
                           double* glam, void* ws, cudaStream_t st);

}  // namespace ptv

// ---- lane-per-fiber streaming engine (kernels_lane.cu): slope-form scan, TMA-tiled windows, no transposed copies ----
namespace ptvl {
enum { LANE_PLAIN = 0, LANE_DR_B = 1, LANE_DR_B_FINAL = 2, LANE_DRA = 3, LANE_DRA_FINAL = 4, LANE_DRB = 5, LANE_PLAIN_T = 6 };      // fused pass arithmetic (PassOp in kernels_lane.cu)
// prox over the fibers (nf, len, inc); returns cudaErrorInvalidConfiguration when the shape does not suit (caller falls back)
template <typename T>
cudaError_t lane_prox(int op, const T* A, const T* B, const T* C, T* X, long long nf, int len, long long inc, T lam, void* scratch,
                      cudaStream_t st, T* X2 = nullptr, const T* lamf = nullptr, long long fpi = 1);   // lamf: per-fiber penalties (plain op), all > 0
void* lane_scratch(long long nf, int len);          // per-device records / counters (allocates: call outside stream capture)
unsigned long long lane_scratch_generation();       // per device: allocations of that buffer so far (its layout changes with each)
bool lane_shape_ok(long long nf, int len, long long inc, size_t elem, const void* const* ptrs, int nptrs);
void lane_set_tuning(int clen, int halo, int variant);
void lane_set_tasklog(unsigned long long* dev, long long cap_tasks);
unsigned long long lane_read_stats(int reset);
}  // namespace ptvl

// ---- backward pass of the batched 1D prox (vjp.cu, contract in vjp_core.cuh) ----
namespace ptvv {
// gx (and gw unless nullptr) from the forward output y and the upstream gradient g over the fibers (nf, len, inc); weights as in
// prox_fibers.  scratch: vjp_scratch_bytes(nf, len) bytes (0: none needed).  Outputs must not overlap inputs.
template <typename T>
cudaError_t vjp_fibers(const T* y, const T* g, T* gx, T* gw, long long nf, int len, long long inc, T lam, const T* lamv, void* scratch,
                       cudaStream_t st);
// The same, with "fused" and the edge signs read from a segmentation tape (vjp_core.cuh) of y instead of y and the weights.
template <typename T>
cudaError_t vjp_fibers_tape(const uint32_t* F, const uint32_t* U, const T* g, T* gx, T* gw, long long nf, int len, long long inc,
                            void* scratch, cudaStream_t st);
// The segmentation tape of y over the fibers (nf, len, inc), nf a multiple of inc: F and U of vjp_tape_set_bytes(nf * len) bytes each.
template <typename T>
cudaError_t fiber_tape(const T* y, long long nf, int len, long long inc, T lam, const T* lamv, uint32_t* F, uint32_t* U, cudaStream_t st);
// The same with fiber j's penalty lamf[j / fpi] (device table; fpi a multiple of inc, so that a group is a range of elements): bit for
// bit the uniform tape of each fiber with its own penalty.
template <typename T>
cudaError_t fiber_tape_lamf(const T* y, long long nf, int len, long long inc, const T* lamf, long long fpi, uint32_t* F, uint32_t* U,
                            cudaStream_t st);
size_t vjp_scratch_bytes(long long nf, int len);
int vjp_chunk_len(long long nf, int len);
void vjp_set_tuning(int clen);
}  // namespace ptvv
