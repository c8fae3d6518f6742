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
                           Engine eng, T* scratch, cudaStream_t st, long long scratch_elems = 0);

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
template <typename T> cudaError_t ew_mean_abs_diff(const T* a, const T* b, long long n, double* scratch, double* result,
                                                   cudaStream_t st);                  // *result = mean|a-b| (device)
template <typename T> cudaError_t ew_pd_combine(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                double* scratch, double* result, cudaStream_t st);
template <typename T> cudaError_t ew_pdr_combine(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                 double* scratch, double* result, cudaStream_t st);
template <typename T> cudaError_t ew_div_scalar(const T* y, T* x, long long n, T k, cudaStream_t st);             // x = y / k
template <typename T> cudaError_t ew_mean_abs_step(const T* y, long long n, double* out, cudaStream_t st);       // out[0] = mean |y[e+1] - y[e]|
template <typename T> cudaError_t ew_dr_first(const T* Y, const T* t, T* U, T* D, long long n, cudaStream_t st);  // D = t - t ; U = Y - (2 D - t)
constexpr int REDUCE_BLOCKS = 1184;    // fixed, not the device's SM count (~9 per SM on a 132-SM H100): partial sums are combined in
                                       // the same fixed order on every GPU (deterministic)

// ---- device-resident solvers (solver.cu).  All arrays are device pointers; `ws` must hold ws_bytes_*() bytes. ----
template <typename T> size_t ws_bytes_dr2(size_t M, size_t N, int batch);
template <typename T> int dr2_device(size_t M, size_t N, int batch, int row_major, const T* Y, T w1, T w2, T* out, int maxit, double* info,
                                     void* ws, Engine eng, cudaStream_t st);
// DR2L1W_TV on one M x N column-major image; W1: (M-1) x N, W2: M x (N-1) column-major; workspace of ws_bytes_dr2(M, N, 1) bytes
template <typename T> int drw_device(size_t M, size_t N, const T* Y, const T* W1, const T* W2, T* out, int maxit, double* info, void* ws,
                                     Engine eng, cudaStream_t st);
template <typename T> size_t ws_bytes_pd(long long n, int npen);
// PD2_TV / PD_TV (proximal Dykstra, stop rule mean|x - x_old| <= STOP_PD).  tape: nullptr, or the recorded forward's buffer (header
// written by the caller after the call, from info[0]): the segmentation tape of every pass
template <typename T> int pd2_device(const T* y, const double* lambdas, const double* dims, T* x, double* info, const int* ns,
                                     int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st, void* tape = nullptr);
template <typename T> int pd_device(const T* y, const double* lambdas_scaled, const double* dims, T* x, double* info,
                                    const int* ns, int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st,
                                    void* tape = nullptr);
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
size_t drw_tape_bytes(size_t M, size_t N, int maxit);                    // header + (2K + 2) passes x two bitsets
template <typename T> size_t ws_bytes_drw_record(size_t M, size_t N);
template <typename T> size_t ws_bytes_drw_vjp(size_t M, size_t N);
// drw_device's iteration with plain prox passes (bit for bit the same output), writing the segmentation tape of every pass.  The
// tape's size (drw_tape_bytes) and the arguments are checked by the caller.
template <typename T> cudaError_t drw_record_device(size_t M, size_t N, const T* Y, const T* W1, const T* W2, T* out, int maxit, void* tape,
                                                    void* ws, Engine eng, cudaStream_t st);
const char* drw_tape_check(const void* tape, size_t elem, size_t M, size_t N, int maxit, cudaStream_t st);
// gY, and per-edge gW1 / gW2 unless nullptr, from the tape alone
template <typename T> cudaError_t drw_vjp_device(size_t M, size_t N, int maxit, const void* tape, const T* gout, T* gY, T* gW1, T* gW2,
                                                 void* ws, cudaStream_t st);

// PDR_TV (src/TVNDopt.cpp:280-500): parallel Douglas-Rachford, fixed iteration count; same workspace as pd_device.  tape: nullptr, or
// the recorded forward's buffer (header written by the caller): the segmentation tape of every pass but the last iteration's
template <typename T> int pdr_device(const T* y, const double* lambdas_scaled, const double* dims, T* x, double* info,
                                     const int* ns, int nds, int npen, int maxIters, void* ws, Engine eng, cudaStream_t st,
                                     void* tape = nullptr);
// the fibers of an n-element column-major array of dims ns[0..nds) along the 1-based axis `dim`; false when dim is not an axis
bool geom_of(const int* ns, int nds, double dim, long long n, FiberGeom* g);
// ---- exact backward pass of PDR_TV (dr2_vjp.cu, DESIGN.md section 13) ----
constexpr int PDR_TAPE_MAX_DIMS = 16;                                    // axes the tape header holds
size_t pdr_tape_bytes(const int* ns, int nds, int npen, int maxIters);    // header + (K - 1) npen passes x two bitsets; 0: too large
// the tape of pass p (output y over the fibers g, penalty lam) into a tape of n-element passes
template <typename T> cudaError_t pdr_tape_pass(void* tape, long long n, long long p, const T* y, FiberGeom g, T lam, cudaStream_t st);
// writes the 256-byte header (arguments checked by the caller; axes = dims - 1)
cudaError_t pdr_tape_header(void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, cudaStream_t st);
// validates a tape's header against the arguments (one stream synchronisation): nullptr ok, else the reason
const char* pdr_tape_check(const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                           cudaStream_t st);
template <typename T> size_t ws_bytes_pdr_vjp(const int* ns, int nds, int npen, const double* dims, bool want_glam);
// gY, and glam[npen] (d/d of the scaled penalties) unless nullptr, from the tape alone; arguments checked by the caller
template <typename T> cudaError_t pdr_vjp_device(const int* ns, int nds, int npen, const double* dims, int maxIters, const void* tape,
                                                 const T* gout, T* gY, double* glam, void* ws, cudaStream_t st);
// ---- exact backward passes of PD_TV and PD2_TV (dr2_vjp.cu, DESIGN.md section 14); pd2 selects PD2_TV ----
// header + the capacity of maxIters (0: 35) iterations: maxIters npen passes (PD_TV), 2 maxIters (PD2_TV; 1 when npen = 1); 0 when
// the byte count does not fit in size_t
size_t pd_tape_bytes(bool pd2, const int* ns, int nds, int npen, int maxIters);
// writes the 256-byte header after the solve: capacity maxIters, iters = the iterations run (info[0])
cudaError_t pd_tape_header(bool pd2, void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters,
                           cudaStream_t st);
const char* pd_tape_check(bool pd2, const void* tape, size_t elem, const int* ns, int nds, int npen, const double* dims, int maxIters,
                          int iters, cudaStream_t st);
// gY, and glam[npen] unless nullptr (PD_TV: d/d of the scaled penalties; PD2_TV: of the penalties as given), from the tape of a solve
// that ran `iters` iterations; arguments checked by the caller; workspace ws_bytes_pdr_vjp
template <typename T> cudaError_t pd_vjp_device(bool pd2, const int* ns, int nds, int npen, const double* dims, int iters, const void* tape,
                                                const T* gout, T* gY, double* glam, void* ws, cudaStream_t st);

}  // namespace ptv

// ---- lane-per-fiber streaming engine (kernels_lane.cu): slope-form scan, TMA-tiled windows, no transposed copies ----
namespace ptvl {
enum { LANE_PLAIN = 0, LANE_DR_B = 1, LANE_DR_B_FINAL = 2, LANE_DRA = 3, LANE_DRA_FINAL = 4, LANE_DRB = 5, LANE_PLAIN_T = 6 };      // fused pass arithmetic (PassOp in kernels_lane.cu)
// prox over the fibers (nf, len, inc); returns cudaErrorInvalidConfiguration when the shape does not suit (caller falls back)
template <typename T>
cudaError_t lane_prox(int op, const T* A, const T* B, const T* C, T* X, long long nf, int len, long long inc, T lam, void* scratch,
                      cudaStream_t st, T* X2 = nullptr);
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
size_t vjp_scratch_bytes(long long nf, int len);
int vjp_chunk_len(long long nf, int len);
void vjp_set_tuning(int clen);
}  // namespace ptvv
