/*
 * proxtv_b200.h -- C ABI of libproxtv_b200.so, the H100-native (sm_90a) TV-L1 proximity operators.
 *
 * Part 1 re-exports, with identical names, prototypes, argument meaning, return values and info[] contents, the hot-path
 * subset of the reference's C interface (src/TVopt.h:88-141 == the cffi cdef in prox_tv/prox_tv_build.py:8-77), so the
 * reference's Python wrapper (prox_tv/__init__.py) or MATLAB mex glue can bind this library instead of its own object
 * code (see INTEGRATION.md).  All pointers in Part 1 are HOST pointers, arrays are float64, 2D/ND arrays column-major;
 * the caller owns every buffer; nothing is retained after return.  The computation runs on the current CUDA device
 * (cuda:0 unless cudaSetDevice was called by the host process); there is no CPU fallback: without a usable device
 * the calls print an error, set info[2] = RC_ERROR (3) where an info array exists and leave the output untouched.
 *
 * Part 2 adds what the BASELINE configurations need and the reference lacks: device-pointer variants (no PCIe traffic),
 * a leading batch dimension, float32 instantiations and pinned-host helpers.
 *
 * Plain C: no C++/torch types cross this boundary.
 */
#ifndef PROXTV_B200_H
#define PROXTV_B200_H
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* info[] slots and return codes -- reference: src/general.h:58-73 */
#define PROXTV_INFO_ITERS 0
#define PROXTV_INFO_GAP 1
#define PROXTV_INFO_RC 2
#define PROXTV_RC_OK 0
#define PROXTV_RC_ITERS 1
#define PROXTV_RC_STUCK 2
#define PROXTV_RC_ERROR 3

/* ------------------------------------------------------------------------------------------------------------------
 * Part 1 -- drop-in symbols (host pointers, float64)
 * ------------------------------------------------------------------------------------------------------------------ */

/* replaces src/TVL1opt_hybridtautstring.cpp:237 (prototype src/TVopt.h:96).  x = argmin 0.5|x-y|^2 + lambda*sum|x_i-x_{i+1}|.
 * Computed with the linearized taut-string scan; the reference's switch to the classic method after n^1.05 steps is an
 * execution-time heuristic that changes results by <= 5e-11 abs and is not reproduced. */
void hybridTautString_TV1(double *y, int n, double lambda, double *x);
/* replaces src/TVL1opt_hybridtautstring.cpp:56 (src/TVopt.h:97); backtracksexp is accepted and ignored (see above). */
void hybridTautString_TV1_custom(double *y, int n, double lambda, double *x, double backtracksexp);
/* replaces src/TVL1opt_tautstring.cpp:355 (src/TVopt.h:95).  Returns 1.  lam <= 0 or n == 1: x = signal (:258-263). */
int classicTautString_TV1(double *signal, int n, double lam, double *prox);
/* replaces src/TVL1opt.cpp:359 (src/TVopt.h:94).  Returns 1.  Bit-identical to the reference. */
int linearizedTautString_TV1(double *y, double lambda, double *x, int n);
/* replaces src/condat_fast_tv.cpp:78 (src/condat_fast_tv.h).  In-place (output == input) allowed; width <= 0 or
 * lambda < 0: nothing is done (:79). */
void TV1D_denoise(double *input, double *output, const int width, const double lambda);
/* replaces src/TVL1Wopt.cpp:364 (src/TVopt.h:103).  lambda has n-1 entries.  Returns 1.  Bit-identical to the reference. */
int tautString_TV1_Weighted(double *y, double *lambda, double *x, int n);
/* The reference's other 1D TV-L1 solvers: projected Newton (src/TVL1opt.cpp:44, src/TVL1Wopt.cpp:36), Condat's taut-string
 * variant (src/condat_fast_tv.cpp:133), Kolmogorov's (src/TVL1opt_kolmogorov.cpp) and Johnson's dynamic programming
 * (src/johnsonRyanTV.cpp).  Same unique minimiser as the functions above (<= 4e-14 apart on random data with the compiled
 * reference; 9e-7 for TV1D_denoise_tautstring, which truncates a slope to float), so they are served by the same exact kernel.
 * info = {0, 0, RC_OK}; sigma and ws are ignored; weighted forms take n-1 weights. */
int PN_TV1(double *y, double lambda, double *x, double *info, int n, double sigma, void *ws);
int PN_TV1_Weighted(double *Y, double *W, double *X, double *info, int n, double sigma, void *ws);
void TV1D_denoise_tautstring(double *input, double *output, int width, const double lambda);
void SolveTVConvexQuadratic_a1_nw(int n, double *b, double w, double *solution);
void SolveTVConvexQuadratic_a1(int n, double *b, double *w, double *solution);
void dp(int n, double *y, double lam, double *beta);
/* replaces src/TVgenopt.cpp:30 (src/TVopt.h:91) for p == 1 only (other norms: prints an error, RC_ERROR, returns 0).
 * ws is ignored (the reference's Python wrapper always passes NULL). */
int TV(double *y, double lambda, double *x, double *info, int n, double p, void *ws);
/* replaces src/TV2Dopt.cpp:352 (src/TVopt.h:128).  M x N column-major; fixed maxit iterations (<= 0: 35) + final
 * projection; info = {maxit, untouched, RC_OK}; returns 0 on success AND on error, like the reference (:440, :372).
 * norm1, norm2 must be 1; nThreads is ignored. */
int DR2_TV(size_t M, size_t N, double *unary, double W1, double W2, double norm1, double norm2, double *s, int nThreads,
           int maxit, double *info);
/* replaces src/TV2DWopt.cpp:46 (src/TVopt.h:116): DR2_TV's iteration with per-edge weights.  unary, s: M x N column-major;
 * W1: (M-1) x N column-major (weights of the edges along columns), W2: M x (N-1) column-major (edges along rows).
 * info = {maxit, untouched, RC_OK}; returns 0 on success AND on error, like the reference (:135, :64-68).  nThreads is
 * ignored.  Fibers of length 1 (M == 1 or N == 1) are left unchanged (the reference reads past an empty weight line). */
int DR2L1W_TV(size_t M, size_t N, double *unary, double *W1, double *W2, double *s, int nThreads, int maxit, double *info);
/* replaces src/TV2Dopt.cpp:587 (src/TVopt.h:129): the 2D TV-L1 prox by Condat's (alg 0), Chambolle-Pock's (alg 1) or the accelerated
 * Chambolle-Pock (alg 2) primal-dual iteration, run until the relative change of X is 0 or maxit iterations (<= 0: 2500).  Y, X: M x N
 * column-major.  Bit for bit the reference's result; info = {iterations run + 1, untouched, RC_OK}; returns 1.  Another alg prints
 * "Condat2_TV: Algorithm parameter has an invalid value", sets info[2] = 3 and returns 0.  M == 1 or N == 1: the missing difference
 * term is left out (the reference reads outside its empty dual array). */
int CondatChambollePock2_TV(size_t M, size_t N, double *Y, double lambda, double *X, short alg, int maxit, double *info);
/* replaces src/TV2Dopt.cpp:59 (src/TVopt.h:126).  npen <= 2, norms must be 1, dims are 1-based; info = {iters, stop, RC};
 * RC_ITERS is set when iters >= 35 regardless of maxIters (:289); returns 1 ok / 0 error. */
int PD2_TV(double *y, double *lambdas, double *norms, double *dims, double *x, double *info, int *ns, int nds, int npen,
           int ncores, int maxIters);
/* replaces src/TVNDopt.cpp:48 (src/TVopt.h:137).  Like the reference it multiplies lambdas[] by npen IN PLACE (:100-101). */
int PD_TV(double *y, double *lambdas, double *norms, double *dims, double *x, double *info, int *ns, int nds, int npen,
          int ncores, int maxIters);
/* replaces src/TVNDopt.cpp:280 (src/TVopt.h:138; reached from MATLAB only in the reference, matlab/solveTVND_PDR.cpp:89): parallel
 * Douglas-Rachford over npen one-dimensional TV-L1 terms.  Runs exactly maxIters iterations (<= 0: 35; the reference's loop has no
 * stop test); multiplies lambdas[] by npen IN PLACE (:339-340); info = {iters, mean|x - x_last| of the last iteration, RC_ITERS when
 * iters >= 35 else RC_OK}; returns 1 ok / 0 error.  norms must be 1 (the reference's p = 2 / general-p terms are out of scope). */
int PDR_TV(double *y, double *lambdas, double *norms, double *dims, double *x, double *info, int *ns, int nds, int npen,
           int ncores, int maxIters);

/* ------------------------------------------------------------------------------------------------------------------
 * Part 2 -- extensions.  *_dev functions take DEVICE pointers and a cudaStream_t passed as void* (NULL = default
 * stream); they run on the CURRENT device (cudaSetDevice), which must own the pointers and the stream -- workspaces, streams and
 * captured graphs are kept per device; they enqueue work and return without synchronising unless stated.  Return value: 1 ok / 0 error, except the
 * DR2 family which follows DR2_TV (always 0; check info[2]).
 * ------------------------------------------------------------------------------------------------------------------ */

int proxtv_device_count(void);                 /* usable CUDA devices (0 => every entry point fails loudly) */
const char *proxtv_last_error(void);           /* last error text of the calling thread ("" if none) */
const char *proxtv_version(void);

/* kernel family / Douglas-Rachford schedule (for measurements and tests).  0 auto: the lane-per-fiber streaming engine in slope
 * form (7) wherever the shape suits TMA tiling (16-byte aligned bases, row pitch a multiple of 16 bytes, positive weights, enough
 * fibers), else the chunked family; 1 sequential lane-per-fiber; 2 chunked speculative scan with the plain serial schedule;
 * 3 chunked with direct strided staging; 4 pipelined gather/scatter schedule; 5 transposeless schedule (scan kernels write both
 * layouts); 6 plain transposes around a fused row kernel; 7 the lane engine (kernels_lane.cu; DR2_TV: column pass over contiguous
 * fibers, row pass with the three operands combined at landing); 8 the lane engine with the transposed DR2_TV schedule (both passes
 * strided, arithmetic in the drains, results written transposed; what row-major images always use).  Engines 2, 4, 5, 6 are
 * bit-identical to each other (the reference's own arithmetic); 7 and 8 are bit-identical to each other and agree with the others to
 * ~1e-13 (same decisions, slope-form arithmetic).  The 1D entry points of Part 1 always use the bit-faithful chunked kernels.
 * Returns the previous value. */
int proxtv_set_engine(int engine);

/* Batched 1D prox over the fibers of a column-major array: nf fibers of len samples, fiber j starting at
 * (j / inc) * inc * len + (j % inc) with element stride inc (the reference's slicing rule, src/TVNDopt.cpp:184-188;
 * inc == 1: nf contiguous signals back to back).  lamv == NULL: uniform weight lam, else per-edge weights laid out the
 * same way with len-1 samples per fiber (batched tautString_TV1_Weighted). */
int proxtv_prox_fibers_dev_f64(const double *in, double *out, long long nf, int len, long long inc, double lam,
                               const double *lamv, void *stream);
int proxtv_prox_fibers_dev_f32(const float *in, float *out, long long nf, int len, long long inc, float lam,
                               const float *lamv, void *stream);
/* Backward pass (vector-Jacobian product) of proxtv_prox_fibers_dev_*: y = the forward's output, g = the upstream gradient, gx = the
 * gradient with respect to the input, all laid out like the fibers; gw (may be NULL) = the gradient with respect to the per-edge
 * weights, laid out like lamv (len-1 samples per fiber; with lamv == NULL its sum over a fiber is the gradient of lam).  Exactly,
 * per fiber, in double and rounded once when stored: edge e is fused iff y[e] == y[e+1] and its weight (lamv[e], or lam) is > 0;
 * every sample gets the mean of g over its run of fused edges, summed left to right from 0.0; gw[e] = sgn(y[e+1] - y[e]) *
 * (gx[e] - gx[e+1]) on unfused edges, +0 on fused ones.  The result does not depend on how the work is split.  Outputs must not
 * overlap inputs (not checked).  Returns 1 ok / 0 error; refused without writing anything: nf < 0, len < 0, inc < 1, y, g or gx
 * NULL, lamv == NULL with lam < 0.  nf == 0 or len == 0: returns 1, does nothing. */
int proxtv_prox_fibers_vjp_dev_f64(const double *y, const double *g, double *gx, double *gw, long long nf, int len, long long inc,
                                   double lam, const double *lamv, void *stream);
int proxtv_prox_fibers_vjp_dev_f32(const float *y, const float *g, float *gx, float *gw, long long nf, int len, long long inc,
                                   float lam, const float *lamv, void *stream);
/* tests: chunk length of the backward pass's work split (0 = automatic; whole fibers when it is >= len) */
void proxtv_vjp_tuning(int chunk_len);
/* Segmentation tape of y (the forward's output) over the fibers (nf, len, inc), nf a multiple of inc: what the backward pass above
 * needs of y, in 2 bits per element.  F and U are bitsets over the nf * len elements in storage order, ceil(nf * len / 32) uint32
 * words each (bit i: word i / 32, bit i % 32), the words up to the next multiple of 256 bytes written as 0.  Bit i describes element
 * i and its successor i + inc along its fiber: (F, U) = (1, 0) fused (equal as stored and weight > 0), (0, 1) the successor is
 * greater, (0, 0) it is smaller -- also every fiber's last sample --, (1, 1) equal with a zero weight (not fused, sign 0).  Refused
 * without writing anything: nf < 0, len < 0, inc < 1, nf not a multiple of inc, y, F or U NULL, lamv == NULL with lam < 0. */
int proxtv_fiber_tape_dev_f64(const double *y, long long nf, int len, long long inc, double lam, const double *lamv, unsigned *F,
                              unsigned *U, void *stream);
int proxtv_fiber_tape_dev_f32(const float *y, long long nf, int len, long long inc, float lam, const float *lamv, unsigned *F,
                              unsigned *U, void *stream);
/* proxtv_prox_fibers_vjp_dev_* driven by a tape instead of (y, lam, lamv): given the tape of (y, lam, lamv), the same gx and gw bit
 * for bit.  Refusals as above (F, U, g or gx NULL; nf not a multiple of inc). */
int proxtv_prox_fibers_vjp_tape_dev_f64(const unsigned *F, const unsigned *U, const double *g, double *gx, double *gw, long long nf,
                                        int len, long long inc, void *stream);
int proxtv_prox_fibers_vjp_tape_dev_f32(const unsigned *F, const unsigned *U, const float *g, float *gx, float *gw, long long nf,
                                        int len, long long inc, void *stream);
/* host-pointer form of the above (pageable or pinned memory); synchronous.  in and out hold nf * len elements, so nf must be a
 * multiple of inc; other geometries are refused (returns 0) without writing anything. */
int proxtv_prox_fibers_f64(const double *in, double *out, long long nf, int len, long long inc, double lam,
                           const double *lamv);
int proxtv_prox_fibers_f32(const float *in, float *out, long long nf, int len, long long inc, float lam,
                           const float *lamv);

/* DR2_TV on `batch` independent M x N images stored back to back.  info (host, 3 doubles, may be NULL).
 * row_major = 0: column-major images (the reference's layout); 1: row-major (C order) images -- the pass order
 * (axis 0 first, then axis 1) is the same, only the kernels' stride roles swap, so no transpose is ever made. */
int proxtv_DR2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, double W1, double W2, double *out, int maxit,
                          double *info, void *stream);
int proxtv_DR2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, float W1, float W2, float *out, int maxit,
                          double *info, void *stream);
/* Exact backward pass of DR2_TV (DESIGN.md section 11).  The gradient is the one of the function computed: the lane engine's fixed
 * schedule of K = maxit iterations (0: 35) and the final projection, every prox pass with the Jacobian of proxtv_prox_fibers_vjp_dev_*.
 * record: DR2_TV as proxtv_DR2_TV_dev_* computes it (bit for bit whenever that call takes a lane schedule; within rounding
 * otherwise), with plain prox passes, writing into the device buffer `tape` (at least proxtv_DR2_TV_tape_bytes() bytes) a 256-byte
 * header and the segmentation tapes (proxtv_fiber_tape_dev_*) of the 2K + 1 passes after the first column pass.  Returns 1 ok / 0
 * error (info[2] = 3 too); refused without writing anything: M, N or batch < 1, Y, out or tape NULL, a negative weight, tape_bytes
 * too small.  vjp: from the tape alone, gY = the gradient with respect to Y for the upstream gradient gout (both laid out like out)
 * and, unless glam is NULL, glam = 2 * batch doubles, per image [W1, W2] -- the gradients of the two penalties.  Deterministic (no
 * atomics); synchronises the stream once (reads the tape's header).  Returns 1 ok / 0 error; refused without writing anything: M, N
 * or batch < 1, tape, gout or gY NULL, a header that does not match the arguments (dtype, shape, batch, row_major, maxit). */
size_t proxtv_DR2_TV_tape_bytes(size_t M, size_t N, int batch, int maxit);
int proxtv_DR2_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, double W1, double W2, double *out,
                                 int maxit, void *tape, size_t tape_bytes, double *info, void *stream);
int proxtv_DR2_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, float W1, float W2, float *out,
                                 int maxit, void *tape, size_t tape_bytes, double *info, void *stream);
int proxtv_DR2_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, int maxit, const void *tape, const double *gout,
                              double *gY, double *glam, void *stream);
int proxtv_DR2_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, int maxit, const void *tape, const float *gout,
                              float *gY, double *glam, void *stream);
int proxtv_DR2_TV_batched_f64(size_t M, size_t N, int batch, const double *Y, double W1, double W2, double *out, int maxit,
                              double *info);
int proxtv_DR2_TV_batched_f32(size_t M, size_t N, int batch, const float *Y, float W1, float W2, float *out, int maxit,
                              double *info);

/* CondatChambollePock2_TV on `batch` independent M x N images stored back to back, column-major (row_major = 0) or C order (1); the
 * same bits in both orders.  Each image runs until its own stop test holds.  info: host, 3 doubles per image ({iterations run + 1,
 * untouched, RC}), may be NULL.  float32: float32 arithmetic, step sizes rounded once from float64, stop sums in float64.  The dev
 * form reads a running-image count back every 64 iterations to end early and synchronises the stream before it returns; the
 * batched form takes host arrays.  Returns 1 ok / 0 error (info[2] = 3 for every image). */
int proxtv_CP2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, double lambda, double *X, int alg, int maxit,
                          double *info, void *stream);
int proxtv_CP2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, double lambda, float *X, int alg, int maxit,
                          double *info, void *stream);
int proxtv_CP2_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double *Y, double lambda, double *X, int alg, int maxit,
                              double *info);
int proxtv_CP2_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float *Y, double lambda, float *X, int alg, int maxit,
                              double *info);
/* The weighted form of proxtv_CP2_TV_* (DESIGN.md section 15.1): the same iteration with each dual clipped to its own edge's weight
 * instead of one lambda -- the converged counterpart of DR2L1W_TV.  W1 weights the edge (i, j)-(i+1, j), W2 the edge (i, j)-(i, j+1);
 * the maps are back to back per image and laid out like proxtv_DR2L1W_TV_batched_*'s (below), in the images' storage order.  With
 * every weight equal to lambda the result is proxtv_CP2_TV_*'s bit for bit; a zero weight disconnects its edge.  Weights must be
 * >= 0 (not checked).  alg 0 (Condat) or 1 (Chambolle-Pock) only: the accelerated rule takes its step sizes from one lambda.
 * Return values, info rows and the float32 rules as proxtv_CP2_TV_*; also refused (info[2] = 3 for every image): alg 2, W1 NULL
 * with M > 1, W2 NULL with N > 1. */
int proxtv_CP2W_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1, const double *W2,
                           double *X, int alg, int maxit, double *info, void *stream);
int proxtv_CP2W_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1, const float *W2,
                           float *X, int alg, int maxit, double *info, void *stream);
int proxtv_CP2W_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1, const double *W2,
                               double *X, int alg, int maxit, double *info);
int proxtv_CP2W_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1, const float *W2,
                               float *X, int alg, int maxit, double *info);
/* Backward pass of the converged solves proxtv_CP2_TV_* / proxtv_CP2W_TV_* (DESIGN.md section 15.2), alg 0 and 1.  It is not the
 * derivative of the iterations computed but the Jacobian of the prox itself at the partition the forward reached, so it is right
 * when the forward has converged.  An edge e = (i, j), j the successor of i along its axis, is FUSED iff its weight w_e (lambda, or its
 * entry of W1 / W2) is > 0 and either |U_e| < w_e for the final dual U_e of the image's last iteration or X_i == X_j as stored; a NaN
 * never fuses.  Clusters are the 4-connected components of the fused edges, per image.
 * record: the _dev_ call, bit for bit the same X and info, then a fused-edge tape into the device buffer `tape` (at least
 * proxtv_CP2_TV_tape_bytes() bytes, the same size for both forms): a 256-byte header (dtype, M, N, batch, row_major, weighted) and
 * two bitsets in storage order (bit q: q fused with its successor along the contiguous axis; along the strided axis), each laid out
 * like proxtv_fiber_tape_dev_*'s.  Returns 1 ok / 0 error (info[2] = 3 for every image); refused without writing anything else: alg
 * 2, an invalid alg, M, N or batch < 1, M N >= 2^31, Y, X, tape (or a needed weight map) NULL, a negative lambda, tape_bytes too
 * small.
 * vjp: from the tape, the recorded result X and the upstream gradient gout (both laid out like X): gY = the cluster means of gout,
 * gY_i = (T)(S_C / |C|) with S_C the sum of (double) gout over i's cluster C; per-edge gW1 / gW2 (weighted form, laid out like W1 / W2,
 * each may be NULL) = (T)(sgn(X_j - X_i) ((double) gY_i - (double) gY_j)) on cut edges and +0 on fused ones; unless glam is NULL,
 * glam = 2 * batch doubles, per image [sum of those edge gradients along axis 0, along axis 1] (the gradient of lambda per axis).
 * Deterministic: S_C is summed exactly in fixed point and rounded once, glam in a fixed order; the same bits in both storage orders.
 * Synchronises the stream once (reads the tape's header).  Returns 1 ok / 0 error; refused without writing anything: M, N or batch <
 * 1, M N >= 2^31, tape, X, gout or gY NULL, a header that does not match the arguments (dtype, shape, batch, row_major, weighted). */
size_t proxtv_CP2_TV_tape_bytes(size_t M, size_t N, int batch);
int proxtv_CP2_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, double lambda, double *X, int alg,
                                 int maxit, double *info, void *tape, size_t tape_bytes, void *stream);
int proxtv_CP2_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, double lambda, float *X, int alg,
                                 int maxit, double *info, void *tape, size_t tape_bytes, void *stream);
int proxtv_CP2W_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1, const double *W2,
                                  double *X, int alg, int maxit, double *info, void *tape, size_t tape_bytes, void *stream);
int proxtv_CP2W_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1, const float *W2,
                                  float *X, int alg, int maxit, double *info, void *tape, size_t tape_bytes, void *stream);
int proxtv_CP2_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, const void *tape, const double *X, const double *gout,
                              double *gY, double *glam, void *stream);
int proxtv_CP2_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, const void *tape, const float *X, const float *gout,
                              float *gY, double *glam, void *stream);
int proxtv_CP2W_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, const void *tape, const double *X, const double *gout,
                               double *gY, double *gW1, double *gW2, double *glam, void *stream);
int proxtv_CP2W_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, const void *tape, const float *X, const float *gout,
                               float *gY, float *gW1, float *gW2, double *glam, void *stream);

/* DR2L1W_TV with device arrays (layouts as above; f32 is an extension the reference lacks). */
int proxtv_DR2L1W_TV_dev_f64(size_t M, size_t N, const double *Y, const double *W1, const double *W2, double *out, int maxit,
                             double *info, void *stream);
int proxtv_DR2L1W_TV_dev_f32(size_t M, size_t N, const float *Y, const float *W1, const float *W2, float *out, int maxit,
                             double *info, void *stream);
/* Exact backward pass of DR2L1W_TV (DESIGN.md section 12): the gradient of the function computed, K = maxit (0: 35) iterations and
 * the final pair, every prox pass with the Jacobian of proxtv_prox_fibers_vjp_dev_*.  Layouts as proxtv_DR2L1W_TV_dev_*.
 * record: proxtv_DR2L1W_TV_dev_* bit for bit, with plain prox passes, writing into the device buffer `tape` (at least
 * proxtv_DR2L1W_TV_tape_bytes() bytes) a 256-byte header and the segmentation tapes (proxtv_fiber_tape_dev_*) of all 2K + 2 passes.
 * Weights must be >= 0 (not checked on the device).  Returns 1 ok / 0 error (info[2] = 3 too); refused without writing anything:
 * M or N < 1, Y, out or tape NULL, W1 NULL with M > 1, W2 NULL with N > 1, tape_bytes too small.  vjp: from the tape alone, gY =
 * the gradient with respect to Y for the upstream gradient gout (both laid out like out) and, unless NULL, gW1 / gW2 = the gradients
 * of the per-edge weights (laid out like W1 / W2; each edge's passes summed in double in backward order, rounded once).
 * Deterministic (no atomics); synchronises the stream once (reads the tape's header).  Returns 1 ok / 0 error; refused without
 * writing anything: M or N < 1, tape, gout or gY NULL, a header that does not match the arguments (dtype, shape, maxit) -- a
 * DR2_TV tape included. */
size_t proxtv_DR2L1W_TV_tape_bytes(size_t M, size_t N, int maxit);
int proxtv_DR2L1W_TV_record_dev_f64(size_t M, size_t N, const double *Y, const double *W1, const double *W2, double *out, int maxit,
                                    void *tape, size_t tape_bytes, double *info, void *stream);
int proxtv_DR2L1W_TV_record_dev_f32(size_t M, size_t N, const float *Y, const float *W1, const float *W2, float *out, int maxit,
                                    void *tape, size_t tape_bytes, double *info, void *stream);
int proxtv_DR2L1W_TV_vjp_dev_f64(size_t M, size_t N, int maxit, const void *tape, const double *gout, double *gY, double *gW1,
                                 double *gW2, void *stream);
int proxtv_DR2L1W_TV_vjp_dev_f32(size_t M, size_t N, int maxit, const void *tape, const float *gout, float *gY, float *gW1,
                                 float *gW2, void *stream);
/* DR2L1W_TV on `batch` independent M x N images stored back to back (image b starts at b M N), each solved with exactly the
 * single-image iteration (its own 2 * mean start value, columns first).  row_major = 0: column-major images, 1: C-ordered images; the
 * weight maps are back to back per image and laid out in the same order:
 *     row_major = 0:  Y[b M N + j M + i]   W1[b (M-1) N + j (M-1) + i]   W2[b M (N-1) + j M + i]
 *     row_major = 1:  Y[b M N + i N + j]   W1[b (M-1) N + i N + j]       W2[b M (N-1) + i (N-1) + j]
 * W1 weights the edge (i, j)-(i+1, j), W2 the edge (i, j)-(i, j+1).  The (1, 0) call is proxtv_DR2L1W_TV_dev_* itself.  Weights
 * must be >= 0 (not checked on the device).
 * dev: returns 0 like DR2L1W_TV (check info[2]); refused (info[2] = 3, nothing written): batch < 0, Y or out NULL, W1 NULL with
 * M > 1, W2 NULL with N > 1.  record / vjp / tape_bytes: as proxtv_DR2L1W_TV_record_dev_* / _vjp_dev_* / _tape_bytes over all
 * batch M N elements in storage order (tape_bytes: 0 for batch < 1); also refused: batch < 1, and a tape whose header does not
 * match dtype, shape, batch, row_major or maxit (a single-image tape included when batch > 1, and a DR2_TV tape).  The gradients
 * are laid out like Y, W1 and W2; the weight gradients are per image and edge, with no sum across images.
 * host form (_batched_f64 / _f32): host arrays, synchronous. */
size_t proxtv_DR2L1W_TV_batched_tape_bytes(size_t M, size_t N, int batch, int maxit);
int proxtv_DR2L1W_TV_batched_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1, const double *W2,
                                     double *out, int maxit, double *info, void *stream);
int proxtv_DR2L1W_TV_batched_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1, const float *W2,
                                     float *out, int maxit, double *info, void *stream);
int proxtv_DR2L1W_TV_batched_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1,
                                            const double *W2, double *out, int maxit, void *tape, size_t tape_bytes, double *info,
                                            void *stream);
int proxtv_DR2L1W_TV_batched_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1,
                                            const float *W2, float *out, int maxit, void *tape, size_t tape_bytes, double *info,
                                            void *stream);
int proxtv_DR2L1W_TV_batched_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, int maxit, const void *tape, const double *gout,
                                         double *gY, double *gW1, double *gW2, void *stream);
int proxtv_DR2L1W_TV_batched_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, int maxit, const void *tape, const float *gout,
                                         float *gY, float *gW1, float *gW2, void *stream);
int proxtv_DR2L1W_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double *Y, const double *W1, const double *W2,
                                 double *out, int maxit, double *info);
int proxtv_DR2L1W_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float *Y, const float *W1, const float *W2,
                                 float *out, int maxit, double *info);

/* PD2_TV / PD_TV with device arrays y, x (lambdas, dims, ns, info stay on the host).  Synchronous (the stop test needs
 * one 8-byte read-back per iteration).  proxtv_PD_TV_* scale lambdas in place like PD_TV. */
int proxtv_PD2_TV_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds,
                          int npen, int maxIters, void *stream);
int proxtv_PD2_TV_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                          int maxIters, void *stream);
int proxtv_PD_TV_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds, int npen,
                         int maxIters, void *stream);
int proxtv_PD_TV_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                         int maxIters, void *stream);
int proxtv_PDR_TV_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds, int npen,
                          int maxIters, void *stream);
int proxtv_PDR_TV_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                          int maxIters, void *stream);
/* Exact backward pass of PDR_TV (DESIGN.md section 13).  The gradient is the one of the function computed: K = maxIters (0: 35)
 * iterations of npen 1D prox passes and one combine, every pass with the Jacobian of proxtv_prox_fibers_vjp_dev_*; the last
 * iteration's passes do not reach x.  tape_bytes: 256 + (K - 1) npen 2 align256(4 ceil(n / 32)) for n = prod ns, 0 for invalid
 * arguments or a size that does not fit in size_t (record refuses that maxIters).  record: the arguments of proxtv_PDR_TV_dev_* plus
 * a device buffer `tape` of at least that many bytes; x and info bit for bit those of proxtv_PDR_TV_dev_* (the same solve, on every
 * engine), lambdas scaled in place like it; writes a 256-byte header and the segmentation tapes (proxtv_fiber_tape_dev_*) of the (K - 1) npen passes that reach x.  Returns 1 ok / 0 error (info[2] = 3
 * too); refused without writing anything, lambdas included: a NULL array, nds outside 1..16, a negative size, npen outside 1..64, a
 * dims entry that is not an axis, a negative penalty, tape_bytes too small.  vjp: from the tape alone, gY = the gradient with respect
 * to y for the upstream gradient gout (both laid out like y) and, unless glam is NULL, glam = npen doubles: the gradients of the
 * SCALED penalties (npen lambdas[i] of the caller; the caller's own penalty gets npen times glam[i]).  Deterministic (no atomics);
 * synchronises the stream once (reads the header).  Returns 1 ok / 0 error; refused without writing anything: NULL arrays, invalid
 * arguments as above, a header that does not match them (dtype, ns, axes, npen, maxIters) -- the tape of any other solver included --
 * and a workspace (about npen + 3 arrays like y, one more with glam) that does not fit in device memory. */
size_t proxtv_PDR_TV_tape_bytes(const int *ns, int nds, int npen, int maxIters);
int proxtv_PDR_TV_record_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds, int npen,
                                 int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PDR_TV_record_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                                 int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PDR_TV_vjp_dev_f64(const int *ns, int nds, int npen, const double *dims, int maxIters, const void *tape, const double *gout,
                              double *gY, double *glam, void *stream);
int proxtv_PDR_TV_vjp_dev_f32(const int *ns, int nds, int npen, const double *dims, int maxIters, const void *tape, const float *gout,
                              float *gY, double *glam, void *stream);
/* Exact backward passes of PD_TV and PD2_TV (DESIGN.md section 14).  The gradient is the one of the function computed: K iterations,
 * K = the count the forward ran (its info[0]); the stop test only picks K, which is locally constant almost everywhere (where a
 * perturbation changes K the map jumps).  Every prox pass has the Jacobian of proxtv_prox_fibers_vjp_dev_*.  tape_bytes: the capacity
 * for maxIters (0: 35) iterations, 256 + P 2 align256(4 ceil(n / 32)) for n = prod ns with P = maxIters npen (PD_TV) or 2 maxIters
 * (PD2_TV; 1 when npen = 1), 0 for invalid arguments or a size that does not fit in size_t (record refuses that maxIters).
 * record: the arguments of proxtv_PD*_TV_dev_* plus a device buffer `tape` of at least that many bytes; x and info bit for bit
 * those of proxtv_PD*_TV_dev_* (the same solve, on every engine); PD_TV scales lambdas in place like its sibling, PD2_TV does not; writes the segmentation tape of every pass and, after the solve, a 256-byte header with
 * the iteration count run.  Returns 1 ok / 0 error (info[2] = 3 too); refused without writing anything, lambdas included: a NULL
 * array, nds outside 1..16, a negative size, npen outside 1..64 (PD_TV) or 1..2 (PD2_TV), a dims entry that is not an axis, a negative
 * penalty, tape_bytes too small.  vjp: iters = the forward's info[0]; from the tape alone, gY = the gradient with respect to y for the
 * upstream gradient gout (both laid out like y) and, unless glam is NULL, glam = npen doubles: PD_TV's are the gradients of the SCALED
 * penalties (the caller's own penalty gets npen times glam[i]), PD2_TV's those of the penalties as given.  Deterministic (no
 * atomics); synchronises the stream once (reads the header).  Returns 1 ok / 0 error; refused without writing anything: NULL arrays,
 * invalid arguments as above, a header that does not match them (dtype, ns, axes, npen, maxIters, iters) -- the tape of any other
 * solver included -- and a workspace (about npen + 3 arrays like y, one more with glam) that does not fit in device memory. */
size_t proxtv_PD_TV_tape_bytes(const int *ns, int nds, int npen, int maxIters);
size_t proxtv_PD2_TV_tape_bytes(const int *ns, int nds, int npen, int maxIters);
int proxtv_PD_TV_record_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds, int npen,
                                int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD_TV_record_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                                int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD2_TV_record_dev_f64(const double *y, double *lambdas, double *dims, double *x, double *info, int *ns, int nds, int npen,
                                 int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD2_TV_record_dev_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                                 int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD_TV_vjp_dev_f64(const int *ns, int nds, int npen, const double *dims, int maxIters, int iters, const void *tape,
                             const double *gout, double *gY, double *glam, void *stream);
int proxtv_PD_TV_vjp_dev_f32(const int *ns, int nds, int npen, const double *dims, int maxIters, int iters, const void *tape,
                             const float *gout, float *gY, double *glam, void *stream);
int proxtv_PD2_TV_vjp_dev_f64(const int *ns, int nds, int npen, const double *dims, int maxIters, int iters, const void *tape,
                              const double *gout, double *gY, double *glam, void *stream);
int proxtv_PD2_TV_vjp_dev_f32(const int *ns, int nds, int npen, const double *dims, int maxIters, int iters, const void *tape,
                              const float *gout, float *gY, double *glam, void *stream);
int proxtv_PD_TV_f32(const float *y, double *lambdas, double *dims, float *x, double *info, int *ns, int nds, int npen,
                     int maxIters);                                          /* host pointers, float32 */

/* Batched PD_TV / PD2_TV (DESIGN.md section 16): `batch` items, each a column-major array of dims ns[0..nds), back to back at stride
 * prod(ns) in y and x; dims are axes of an item.  Every item runs its own loop and stop rule (PD_TV: while stop_b > 1e-6 and it < maxIters;
 * PD2_TV: the same, and one iteration only when npen = 1), and info[3 b .. 3 b + 2] = [K_b, stop_b, RC_b] as the single-item call gives
 * it.  Under the seq and chunked engines every item's x and info row equal proxtv_PD*_TV_dev_* on that item (into an aligned buffer)
 * bit for bit, whatever batch is and wherever the item sits; under auto / lane the engine is picked for the whole batch.  An item that
 * has stopped costs no more prox work.  lambdas are the penalties as given (PD_TV applies its factor npen to a copy) and are never
 * written.  Same refusals, in the same order, as the single-item entry points, plus batch < 1; a refusal writes nothing but
 * info[3 b + 2] = 3 for every item, and returns 0.  The dev and record entries read the stop values back once per iteration.
 * tape_bytes: nd_head + P 2 align256(4 ceil(n batch / 32)), nd_head = 256 + align256(4 batch), P as for the single-item tape, in 64-bit
 * arithmetic, 0 for invalid arguments or a size that does not fit.  The tape carries its own magic (neither the single-item tapes nor
 * the other solver's are accepted), batch, and each item's K.  vjp: from the tape alone (one stream synchronisation reads its header
 * and K table), gY of every item bit for bit the single-item vjp's for that item's K; glam unless NULL: batch x npen doubles, the
 * gradients of the penalties AS GIVEN for both solvers. */
size_t proxtv_PD_TV_batched_tape_bytes(const int *ns, int nds, int npen, int batch, int maxIters);
size_t proxtv_PD2_TV_batched_tape_bytes(const int *ns, int nds, int npen, int batch, int maxIters);
int proxtv_PD_TV_batched_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds,
                              int npen, int batch, int maxIters, void *stream);
int proxtv_PD_TV_batched_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds, int npen,
                          int batch, int maxIters);                 /* host pointers */
int proxtv_PD_TV_batched_record_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns,
                                     int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD_TV_batched_vjp_dev_f64(const int *ns, int nds, int npen, const double *dims, int batch, int maxIters, const void *tape,
                                  const double *gout, double *gY, double *glam, void *stream);
int proxtv_PD_TV_batched_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds,
                              int npen, int batch, int maxIters, void *stream);
int proxtv_PD_TV_batched_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds, int npen,
                          int batch, int maxIters);                 /* host pointers */
int proxtv_PD_TV_batched_record_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns,
                                     int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD_TV_batched_vjp_dev_f32(const int *ns, int nds, int npen, const double *dims, int batch, int maxIters, const void *tape,
                                  const float *gout, float *gY, double *glam, void *stream);
int proxtv_PD2_TV_batched_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds,
                              int npen, int batch, int maxIters, void *stream);
int proxtv_PD2_TV_batched_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds, int npen,
                          int batch, int maxIters);                 /* host pointers */
int proxtv_PD2_TV_batched_record_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns,
                                     int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD2_TV_batched_vjp_dev_f64(const int *ns, int nds, int npen, const double *dims, int batch, int maxIters, const void *tape,
                                  const double *gout, double *gY, double *glam, void *stream);
int proxtv_PD2_TV_batched_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds,
                              int npen, int batch, int maxIters, void *stream);
int proxtv_PD2_TV_batched_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds, int npen,
                          int batch, int maxIters);                 /* host pointers */
int proxtv_PD2_TV_batched_record_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns,
                                     int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes, void *stream);
int proxtv_PD2_TV_batched_vjp_dev_f32(const int *ns, int nds, int npen, const double *dims, int batch, int maxIters, const void *tape,
                                  const float *gout, float *gY, double *glam, void *stream);

/* Per-item penalties (DESIGN.md section 16.1): the _batched_ entry points above with `lambdas` holding batch x npen doubles, item-major --
 * item b's penalties in dims order at lambdas + b npen, as given (PD_TV applies its factor npen to a copy of each row; lambdas is never
 * written).  Item b is solved as the single-item call with its own row solves it: under the seq and chunked engines its x and info row
 * equal proxtv_PD*_TV_dev_* on that item with that row (into an aligned buffer) bit for bit; under auto / lane the engine is picked for
 * the whole batch (the lane guard looks at the largest penalty of the table).  A pass whose running items all have the same penalty for
 * its term runs the kernels of the shared-row call, so equal rows give the _batched_ call's result and info bit for bit on every engine.
 * The record form writes an ordinary batched tape (same size, same format): proxtv_PD*_TV_batched_vjp_dev_* reads it, and its glam rows
 * are the gradients of each item's own penalties as given.  Refusals: those of the _batched_ counterpart in the same order, plus lambdas
 * == NULL; the record form refuses a negative penalty anywhere in the table. */
int proxtv_PD_TV_batched_items_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns,
                                       int nds, int npen, int batch, int maxIters, void *stream);
int proxtv_PD_TV_batched_items_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds,
                                   int npen, int batch, int maxIters);                 /* host pointers */
int proxtv_PD_TV_batched_items_record_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info,
                                              const int *ns, int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes,
                                              void *stream);
int proxtv_PD_TV_batched_items_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns,
                                       int nds, int npen, int batch, int maxIters, void *stream);
int proxtv_PD_TV_batched_items_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds,
                                   int npen, int batch, int maxIters);                 /* host pointers */
int proxtv_PD_TV_batched_items_record_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info,
                                              const int *ns, int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes,
                                              void *stream);
int proxtv_PD2_TV_batched_items_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns,
                                        int nds, int npen, int batch, int maxIters, void *stream);
int proxtv_PD2_TV_batched_items_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info, const int *ns, int nds,
                                    int npen, int batch, int maxIters);                /* host pointers */
int proxtv_PD2_TV_batched_items_record_dev_f64(const double *y, const double *lambdas, const double *dims, double *x, double *info,
                                               const int *ns, int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes,
                                               void *stream);
int proxtv_PD2_TV_batched_items_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns,
                                        int nds, int npen, int batch, int maxIters, void *stream);
int proxtv_PD2_TV_batched_items_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info, const int *ns, int nds,
                                    int npen, int batch, int maxIters);                /* host pointers */
int proxtv_PD2_TV_batched_items_record_dev_f32(const float *y, const double *lambdas, const double *dims, float *x, double *info,
                                               const int *ns, int nds, int npen, int batch, int maxIters, void *tape, size_t tape_bytes,
                                               void *stream);

/* Launch accounting and optional CUDA-event timing per kernel class (0: prox over contiguous fibers, 1: prox over strided
 * fibers, 2: elementwise/reduction helpers).  Launch counters always run; event timing only while enabled.  read():
 * arrays of 3; ms = summed event time, launches = kernels launched, spans = timed brackets; synchronises the events. */
void proxtv_profile_enable(int on);
void proxtv_profile_reset(void);
void proxtv_profile_read(double *ms, long long *launches, long long *spans);

/* pinned host memory for the end-to-end path (cudaHostAlloc / cudaFreeHost) */
void *proxtv_host_alloc(size_t bytes);
void proxtv_host_free(void *p);
/* release the cached device workspace */
void proxtv_release_workspace(void);

/* Lane engine, one batched prox pass with the fused arithmetic `op` over the fibers (nf, len, inc) as above (inc == 1 only with op 0);
 * used by the multi-GPU driver (proxtv_b200/distributed.py) and by the measurement tools.  With x = prox(scan input):
 *   0 plain                 X = prox(A)
 *   1 DR second half        X = (C - B) + prox(A - (2 (C - B) - C))                 (operands combined when their tiles land)
 *   2 DR final projection   X = prox(A - (C - B))
 *   3 DR first half, T      x = prox(A); d = C - x; X^T = B - (2 d - C); X2^T = d   (operands read in the drain; ^T: results written
 *   4 DR final, T           X^T = B - (C - prox(A))                                  fiber-major, element (fiber f, row r) at f * len + r)
 *   5 DR second half, T     X^T = B + prox(A)
 *   6 plain, T              X^T = prox(A)
 * Returns 0 when the shape does not suit the engine (bases and row pitch multiples of 16 bytes).  tuning: chunk length (0 = automatic),
 * halo rows, kernel variant (-1 = default per storage type); stats: fibers that went through the repair path since the last reset. */
int proxtv_lane_prox_dev_f64(int op, const double *A, const double *B, const double *C, double *X, long long nf, int len,
                             long long inc, double lam, void *stream);
int proxtv_lane_prox_dev_f32(int op, const float *A, const float *B, const float *C, float *X, long long nf, int len,
                             long long inc, float lam, void *stream);
/* The batched 1D prox above (plain, unweighted) with one penalty per group of fpi fibers: fiber j's penalty is lamf[j / fpi], lamf a
 * device array of nf / fpi values.  Honours proxtv_set_engine; every fiber's result equals, bit for bit, the uniform pass with its own
 * penalty on the kernel family that ran it (seq and chunked: the reference's linearized taut string; lane: the slope-form scan).  The
 * lane engine takes a table only when every entry is > 0 (the call reads the table back once to know, and to give auto's lane guard
 * its largest entry); a table with a zero runs on the chunked kernels.  Refused without writing anything: fpi < 1, nf not a multiple
 * of fpi, lamf NULL, nf < 0, len < 0, inc < 1.  The tape form: proxtv_fiber_tape_dev_* with fiber j's penalty lamf[j / fpi] (an edge
 * is fused only where its fiber's penalty is > 0), bit for bit the uniform tape of each fiber with its own penalty; refusals of
 * proxtv_fiber_tape_dev_* (lamf in place of the penalty), then fpi < 1, nf not a multiple of fpi, fpi not a multiple of inc. */
int proxtv_prox_fibers_lamf_dev_f64(const double *in, double *out, long long nf, int len, long long inc, const double *lamf, long long fpi,
                                    void *stream);
int proxtv_prox_fibers_lamf_dev_f32(const float *in, float *out, long long nf, int len, long long inc, const float *lamf, long long fpi,
                                    void *stream);
int proxtv_fiber_tape_lamf_dev_f64(const double *y, long long nf, int len, long long inc, const double *lamf, long long fpi, unsigned *F,
                                   unsigned *U, void *stream);
int proxtv_fiber_tape_lamf_dev_f32(const float *y, long long nf, int len, long long inc, const float *lamf, long long fpi, unsigned *F,
                                   unsigned *U, void *stream);
/* same with a second result array (the ops that write two results: 3 = first half of a Douglas-Rachford iteration, transposed) */
int proxtv_lane_prox2_dev_f64(int op, const double *A, const double *B, const double *C, double *X, double *X2, long long nf, int len,
                              long long inc, double lam, void *stream);
void proxtv_lane_tuning(int clen, int halo, int variant);
unsigned long long proxtv_lane_stats(int reset);
/* Under engine 0 (auto) the solvers use the lane engine only while the data keeps segments short -- penalty not larger than about the
 * mean step |y[i+1] - y[i]| of (a sample of) the input, measured with one small kernel and one stream synchronisation per call --
 * and the chunked engine otherwise.  Last decision on the current device: 1 lane, 0 chunked, -1 none taken. */
int proxtv_lane_guard_last(void);
/* tests: contiguous unweighted fibers longer than shared memory go through overlapping tiles whose stitching is verified on the device,
 * and the whole call falls back to the sequential kernel when a check fails.  What the latest proxtv_prox_fibers_* call (or 1D entry
 * point of Part 1) on the current device did: 1 used the tiles, 0 tried them and fell back, -1 did not try them. */
int proxtv_long_fiber_last(void);
/* tools: device buffer of 16 x cap_tasks uint64 that receives, per warp task of the next lane launches (a launch with more tasks than
 * cap_tasks is not logged):
 *   [0] start ns  [1] scan end ns  [2] end ns (globaltimer)  [3] SM id
 *   [4] epochs  [5] scan steps  [6] epochs of fewer than 8 steps (every lane near the landed rows)  [7] waits for a tile
 *   [8] SM cycles (clock64) in the epoch loop, of which  [9] blocked on a tile  [10] other epochs where no lane could move (tail,
 *   retirement)  [11] sweep and drain (including the drain's operand loads)  [12] feed (tile requests, landing)  [13] scan
 *   (the remainder is the epochs' warp reductions)
 *   [14] rows the task scans (owned + halo)  [15] 0
 * NULL switches the log off. */
void proxtv_lane_tasklog(unsigned long long *dev, long long cap_tasks);

#ifdef __cplusplus
}
#endif
#endif /* PROXTV_B200_H */
