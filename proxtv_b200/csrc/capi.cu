// capi.cu -- the extern "C" boundary of libproxtv_b200.so (declared in include/proxtv_b200.h).
//
// Host-pointer entry points stage their arrays through a cached device arena (grow-only; one per process, guarded by a
// mutex), run the device-resident solver and copy the result back.  There is no CPU fallback: if no CUDA device is usable
// every entry point fails loudly.  Error behaviour follows the reference: "<fn>: <msg>" on stdout, info[RC] = RC_ERROR,
// return 0 (src/TV2Dopt.cpp:78-82,368-372).
#include "../../include/proxtv_b200.h"
#include "ptv_internal.h"
#include <limits.h>
#include <mutex>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>

using namespace ptv;

namespace {

thread_local std::string g_err;
std::recursive_mutex g_mu;
int g_engine = ENGINE_AUTO;

struct Arena {
    void* p = nullptr; size_t cap = 0;
    void* get(size_t bytes) {
        if (bytes <= cap) return p;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        size_t want = bytes + (bytes >> 3);
        if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); p = nullptr;
            if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); p = nullptr; cap = 0; return nullptr; }
            cap = bytes; return p; }
        cap = want; return p;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
// solver workspace ; staging of host arrays -- one pair per device, so that a process that works on several devices in turn
// (torch tensors on cuda:0 and cuda:1) never hands one device's memory to kernels running on another
Arena g_ws_d[MAX_DEVICES], g_io_d[MAX_DEVICES];
// the current device's workspace of at least `bytes`; nullptr ("out of memory") when it cannot be had
void* ws_get(size_t bytes) { const int d = device_slot(); return d < 0 ? nullptr : g_ws_d[d].get(bytes); }

// The workspaces, pipeline streams and captured graphs are one set per device, shared by every call: calls are serialised on the
// host by g_mu, and ON THE DEVICE by a per-device event -- a call's stream first waits for the previous call's work (which may
// have been enqueued on another stream), and records the event when its own work is enqueued.  Held for the whole call.
struct WsGuard {
    std::lock_guard<std::recursive_mutex> lk;
    cudaStream_t st; int dev;
    static cudaEvent_t& ev(int d) { static cudaEvent_t e[MAX_DEVICES] = {}; return e[d]; }
    explicit WsGuard(cudaStream_t s) : lk(g_mu), st(s), dev(device_slot()) {
        if (dev < 0) return;
        if (!ev(dev)) { if (cudaEventCreateWithFlags(&ev(dev), cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); ev(dev) = nullptr; dev = -1; } }
        else cudaStreamWaitEvent(st, ev(dev), 0);
    }
    ~WsGuard() { if (dev >= 0 && ev(dev)) cudaEventRecord(ev(dev), st); }
};

// How entry point fn refuses a call: "<fn>: <msg>" becomes proxtv_last_error() and a line on stdout, and info[3 b + RC] = RC_ERROR
// for the first `rows` rows of info (0, 1, or one per item of a batch).  Each refusal returns 0, the entry points' failure value.
struct Refuse {
    const char* fn;
    double* info = nullptr;
    int rows = 0;
    void note(const char* msg) const { g_err = std::string(fn) + ": " + msg; }      // proxtv_last_error() alone
    int mark() const { if (info) for (int b = 0; b < rows; b++) info[3 * (size_t)b + INFO_RC] = RC_ERROR; return 0; }
    int operator()(const char* msg) const { note(msg); printf("%s: %s\n", fn, msg); fflush(stdout); return mark(); }
    // true for cudaSuccess; else refuses with the CUDA error
    bool cuda_ok(cudaError_t e) const {
        if (e == cudaSuccess) return true;
        cudaGetLastError();
        (*this)((std::string("CUDA error: ") + cudaGetErrorString(e)).c_str());
        return false;
    }
    bool have_device() const {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n <= 0) { cudaGetLastError(); (*this)("no usable CUDA device (libproxtv_b200 has no CPU fallback)"); return false; }
        int d = -1;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= MAX_DEVICES - 1) { cudaGetLastError();
            (*this)("current CUDA device index out of the supported range (0..62)"); return false; }
        return true;
    }
};
inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

// The host arrays of one call, staged through the current device's g_io arena on the call's stream.  in() and out() list them;
// stage() gives each an al()-aligned device buffer (8 bytes longer than the array, so an empty one still has its own), points the
// listed pointer at it and copies the inputs in; finish() copies the outputs back and synchronises the stream (nothing listed:
// nothing to do).  Empty arrays are not copied.
template <typename T>
class HostIO {
public:
    HostIO(const Refuse& no, cudaStream_t st) : no_(no), st_(st) {}
    void in(const T*& p, size_t n) { a_[k_++] = Arr{&p, nullptr, p, nullptr, n}; }
    void out(T*& p, size_t n) { a_[k_++] = Arr{nullptr, &p, nullptr, p, n}; }
    bool stage(const char* oom = "out of memory") {
        size_t bytes = 0;
        for (int i = 0; i < k_; i++) bytes += al(a_[i].n * sizeof(T) + 8);
        const int d = device_slot();
        char* p = d < 0 ? nullptr : (char*)g_io_d[d].get(bytes);
        if (!p) return no_(oom);
        for (int i = 0; i < k_; i++) {
            Arr& a = a_[i];
            a.dev = (T*)p; p += al(a.n * sizeof(T) + 8);
            if (a.out) { *a.out = a.dev; continue; }
            *a.in = a.dev;
            if (a.n && !no_.cuda_ok(cudaMemcpyAsync(a.dev, a.from, a.n * sizeof(T), cudaMemcpyHostToDevice, st_))) return false;
        }
        return true;
    }
    bool finish() {
        if (!k_) return true;
        for (int i = 0; i < k_; i++) {
            const Arr& a = a_[i];
            if (a.out && a.n && !no_.cuda_ok(cudaMemcpyAsync(a.to, a.dev, a.n * sizeof(T), cudaMemcpyDeviceToHost, st_))) return false;
        }
        return no_.cuda_ok(cudaStreamSynchronize(st_));
    }
private:
    struct Arr { const T** in; T** out; const T* from; T* to; size_t n; T* dev = nullptr; };
    const Refuse& no_;
    cudaStream_t st_;
    Arr a_[4];
    int k_ = 0;
};

// The batched 1D prox over the fibers (nf, len, inc).  host_io: in, out and lamv are host arrays, staged as nf * len elements (and
// nf * (len - 1) weights) -- with inc > 1 that is the whole slicing only when nf is a multiple of inc (the last fibers of a partial
// slab would lie beyond it).
template <typename T>
int run_prox_fibers(const char* fn, bool host_io, const T* in, T* out, long long nf, int len, long long inc, T lam, const T* lamv,
                    cudaStream_t st) {
    const Refuse no{fn};
    if (host_io && (nf <= 0 || len <= 0)) return 1;
    if (host_io && (inc < 1 || (inc > 1 && nf % inc != 0))) return no("invalid fiber geometry (need inc >= 1 and nf a multiple of inc)");
    if (!no.have_device()) return 0;
    WsGuard guard(st);
    HostIO<T> io(no, st);
    if (host_io) {
        io.in(in, (size_t)nf * len);
        if (lamv) io.in(lamv, (size_t)nf * (len - 1));
        io.out(out, (size_t)nf * len);
    }
    // scratch: staging of strided fibers, or the overlapping tiles of plain contiguous fibers longer than shared memory
    const long long se = nf <= 0 || len <= 0 ? 0 : inc != 1 ? strided_scratch_elems(nf, len) : len > 16384 && !lamv ? lf_scratch_elems(nf, len) : 0;
    T* scr = se ? (T*)ws_get(al((size_t)se * sizeof(T)) + (inc == 1 ? 256 : 0)) : nullptr;
    if (host_io && !io.stage("out of device memory")) return 0;
    long_fiber_note(-1);
    const Engine eng = (!lamv && nf >= 1024 && len >= 64) ? lane_guard<T>((Engine)g_engine, in, nf * (long long)len, (double)lam, st) : (Engine)g_engine;
    if (!no.cuda_ok(prox_fibers<T>(in, nullptr, IN_A, out, 0, FiberGeom{nf, len, inc}, lam, lamv, eng, scr, st, se))) return 0;
    return io.finish() ? 1 : 0;
}

// DR2_TV with host (host_io) or device arrays: `batch` images back to back, column-major (row_major = 0) or C order (1).  Returns 0
// like the reference; with host arrays an empty image reports the iterations the reference would have run (TV2Dopt.cpp:387).
template <typename T>
int run_dr2(const char* fn, bool host_io, size_t M, size_t N, int batch, int row_major, const T* Y, T W1, T W2, T* out, int maxit,
            double* info, cudaStream_t st) {
    const Refuse no{fn, info, 1};
    if (!no.have_device()) return 0;
    WsGuard guard(st);
    const size_t n = M * N * (size_t)batch;
    if (host_io && n == 0) { if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; } return 0; }
    void* ws = ws_get(ws_bytes_dr2<T>(M, N, batch));
    if (!ws) return no("out of memory");                                             // TV2Dopt.cpp:383-384
    if (!host_io) return dr2_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, info, ws, (Engine)g_engine, st);
    HostIO<T> io(no, st);
    io.in(Y, n); io.out(out, n);
    if (!io.stage()) return 0;
    double linfo[3] = {0, 0, RC_OK};                   // a NULL info must not hide a failed solve (nothing is copied back then)
    double* pinfo = info ? info : linfo;
    dr2_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, pinfo, ws, (Engine)g_engine, st);
    if (pinfo[INFO_RC] == RC_ERROR) return no("device solver failed");
    io.finish();
    return 0;
}

// DR2L1W_TV with host (host_io) or device arrays: `batch` images back to back, column-major (row_major = 0) or C order (1); W1:
// (M-1) x N, W2: M x (N-1) per image, laid out like Y (include/proxtv_b200.h).
template <typename T>
int run_drw(const char* fn, bool host_io, size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit,
            double* info, cudaStream_t st) {
    const Refuse no{fn, info, 1};
    if (batch < 0) return no("invalid shape (need batch >= 0)");
    if (!no.have_device()) return 0;
    WsGuard guard(st);
    const size_t n = M * N * (size_t)batch, n1 = M ? (M - 1) * N * (size_t)batch : 0, n2 = N ? M * (N - 1) * (size_t)batch : 0;
    if (n == 0) { if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; } return 0; }
    if (!Y || !out || (n1 && !W1) || (n2 && !W2)) return no("NULL array");
    void* ws = ws_get(ws_bytes_dr2<T>(M, N, batch));
    if (!ws) return no("out of memory");                                             // TV2DWopt.cpp:78-79
    if (!host_io) return drw_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, info, ws, (Engine)g_engine, st);
    HostIO<T> io(no, st);
    io.in(Y, n); io.in(W1, n1); io.in(W2, n2); io.out(out, n);
    if (!io.stage()) return 0;
    double linfo[3] = {0, 0, RC_OK};
    double* pinfo = info ? info : linfo;
    drw_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, pinfo, ws, (Engine)g_engine, st);
    if (pinfo[INFO_RC] == RC_ERROR) return no("device solver failed");
    io.finish();
    return 0;
}

// CondatChambollePock2_TV with host (host_io) or device arrays: `batch` images back to back, column-major (row_major = 0) or C order
// (1); info: host, 3 doubles per image, or NULL.  Returns 1 on success, 0 on failure (src/TV2Dopt.cpp:600-602, :750-756).  A
// refusal marks every image's row (the first one when batch < 1).  weighted (DESIGN.md section 15.1): per-edge maps W1, W2 laid out
// like run_drw's instead of lambda, alg 0 or 1.
template <typename T>
int run_cp2(const char* fn, bool host_io, size_t M, size_t N, int batch, int row_major, const T* Y, double lambda, bool weighted,
            const T* W1, const T* W2, T* X, int alg, int maxit, double* info, cudaStream_t st, void* tape = nullptr) {
    const Refuse no{fn, info, batch > 1 ? batch : 1};
    if (weighted && alg == 2) return no("the weighted solver has no accelerated variant (alg 2); use alg 0 or 1");
    if (alg != 0 && alg != 1 && alg != 2) return no("Algorithm parameter has an invalid value");
    if (batch < 0) return no("invalid shape (need batch >= 0)");
    if (batch == 0) return 1;
    if (M < 1 || N < 1 || M > 0x7fffffff || N > 0x7fffffff) return no("invalid shape (need 1 <= M, N < 2^31)");
    if (!Y || !X || (weighted && ((M > 1 && !W1) || (N > 1 && !W2)))) return no("NULL array");
    if (!no.have_device()) return 0;
    WsGuard guard(st);
    const size_t n = M * N * (size_t)batch;
    void* ws = ws_get(ws_bytes_cp2(M, N, batch, sizeof(T)));
    if (!ws) return no("out of memory");
    HostIO<T> io(no, st);
    if (host_io) {
        io.in(Y, n);
        if (weighted) { io.in(W1, (M - 1) * N * (size_t)batch); io.in(W2, M * (N - 1) * (size_t)batch); }
        io.out(X, n);
        if (!io.stage()) return 0;
    }
    std::vector<int> iters(info ? batch : 0);
    if (!no.cuda_ok(cp2_device<T>(M, N, batch, row_major, Y, lambda, weighted, W1, W2, X, alg, maxit, info ? iters.data() : nullptr, ws, st,
                                  tape)))
        return 0;
    if (!io.finish()) return 0;
    if (info) for (int b = 0; b < batch; b++) { info[3 * (size_t)b + INFO_ITERS] = iters[b]; info[3 * (size_t)b + INFO_RC] = RC_OK; }
    return 1;
}

// The recorded converged solve: run_cp2's device call, then the fused-edge tape (DESIGN.md section 15.2).  Its own refusals come first.
template <typename T>
static int dev_cp2_record(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, double lambda, bool weighted, const T* W1,
                          const T* W2, T* X, int alg, int maxit, double* info, void* tape, size_t tape_bytes, void* stream) {
    const Refuse no{fn, info, batch > 1 ? batch : 1};
    if (alg == 2) return no("the accelerated solver (alg 2) has no converged backward: it does not reach the prox's partition; record with alg 0 or 1");
    if (alg != 0 && alg != 1) return no("Algorithm parameter has an invalid value");
    if (M < 1 || N < 1 || batch < 1 || M > (size_t)INT_MAX || N > (size_t)INT_MAX || M * N > (size_t)INT_MAX)
        return no("invalid shape (need M, N, batch >= 1 and M N < 2^31)");
    if (!Y || !X || !tape || (weighted && ((M > 1 && !W1) || (N > 1 && !W2)))) return no("NULL array");
    if (!weighted && !(lambda >= 0)) return no("negative penalty");
    if (tape_bytes < cp2_tape_bytes(M, N, batch)) return no("tape_bytes smaller than proxtv_CP2_TV_tape_bytes()");
    return run_cp2<T>(fn, false, M, N, batch, row_major, Y, lambda, weighted, W1, W2, X, alg, maxit, info, (cudaStream_t)stream, tape);
}

template <typename T>
static int dev_cp2_vjp(const char* fn, bool weighted, size_t M, size_t N, int batch, int row_major, const void* tape, const T* X, const T* gout,
                       T* gY, T* gW1, T* gW2, double* glam, void* stream) {
    const Refuse no{fn};
    if (M < 1 || N < 1 || batch < 1 || M > (size_t)INT_MAX || N > (size_t)INT_MAX || M * N > (size_t)INT_MAX)
        return no("invalid shape (need M, N, batch >= 1 and M N < 2^31)");
    if (!tape || !X || !gout || !gY) return no("NULL array");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = cp2_tape_check(tape, sizeof(T), M, N, batch, row_major, weighted, (cudaStream_t)stream)) return no(why);
    void* ws = ws_get(ws_bytes_cp2_vjp(M, N, batch));
    if (!ws) return no("out of memory");
    return no.cuda_ok(cp2_vjp_device<T>(M, N, batch, row_major, tape, X, gout, gY, gW1, gW2, glam, ws, (cudaStream_t)stream));
}

// PD_TV and PDR_TV multiply the caller's penalties by the number of terms, in place (TVNDopt.cpp:100-101, :339-340); PD2_TV takes
// them as given.
void scale_penalties(NdSolver s, double* lambdas, int npen) {
    if (s != ND_PD2) for (int i = 0; i < npen; i++) lambdas[i] *= npen;
}

// The device solver of s (solver.cu); tape: nullptr, or the recorded forward's buffer.
template <typename T>
int nd_solve(NdSolver s, const T* y, const double* lambdas, const double* dims, T* x, double* info, const int* ns, int nds, int npen,
             int maxIters, void* ws, cudaStream_t st, void* tape) {
    switch (s) {
    case ND_PD2: return pd2_device<T>(y, lambdas, dims, x, info, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape);
    case ND_PD: return pd_device<T>(y, lambdas, dims, x, info, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape);
    default: return pdr_device<T>(y, lambdas, dims, x, info, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape);
    }
}

// y/x host (host_io) or device pointers.
template <typename T>
int run_pd(const char* fn, NdSolver s, bool host_io, const T* y, double* lambdas, double* norms, double* dims, T* x, double* info,
           int* ns, int nds, int npen, int maxIters, cudaStream_t st) {
    const Refuse no{fn, info, 1};
    if (!no.have_device()) return 0;
    if (norms) for (int i = 0; i < npen; i++) if (norms[i] != 1.0) return no("only p = 1 (TV-L1) penalty terms are implemented on the GPU path");
    if (nds <= 0 || !ns) return no("invalid dimensions");
    NdTerms t;
    nd_terms(ns, nds, 0, nullptr, &t);                 // the element count; the solver checks the terms
    const long long n = t.n;
    WsGuard guard(st);
    scale_penalties(s, lambdas, npen);
    void* ws = ws_get(ws_bytes_pd<T>(n, npen));
    if (!ws) return no("out of memory");
    HostIO<T> io(no, st);
    if (host_io && n > 0) {
        io.in(y, (size_t)n); io.out(x, (size_t)n);
        if (!io.stage()) return 0;
    }
    if (!nd_solve<T>(s, y, lambdas, dims, x, info, ns, nds, npen, maxIters, ws, st, nullptr)) return 0;
    return io.finish() ? 1 : 0;
}

// Backward pass of proxtv_prox_fibers_dev_*: refused calls write nothing; the scratch (chunked work only) comes from the workspace.
template <typename T>
static int dev_vjp(const char* fn, const T* y, const T* g, T* gx, T* gw, long long nf, int len, long long inc, T lam, const T* lamv,
                   void* stream) {
    const Refuse no{fn};
    if (nf < 0 || len < 0 || inc < 1) return no("invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1)");
    if (nf == 0 || len == 0) return 1;
    if (!y || !g || !gx) return no("NULL array");
    if (!lamv && !(lam >= 0)) return no("negative penalty");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    const size_t sb = ptvv::vjp_scratch_bytes(nf, len);
    void* scr = sb ? ws_get(sb) : nullptr;
    if (sb && !scr) return no("out of device memory");
    return no.cuda_ok(ptvv::vjp_fibers<T>(y, g, gx, gw, nf, len, inc, lam, lamv, scr, (cudaStream_t)stream));
}

// The batched 1D prox with fiber j's penalty lamf[j / fpi] (device table); refused calls write nothing.
template <typename T>
static int dev_prox_fibers_lamf(const char* fn, const T* in, T* out, long long nf, int len, long long inc, const T* lamf, long long fpi,
                                void* stream) {
    const Refuse no{fn};
    if (fpi < 1 || nf % fpi != 0) return no("invalid penalty groups (need fpi >= 1 and nf a multiple of fpi)");
    if (!lamf) return no("NULL array");
    if (nf < 0 || len < 0 || inc < 1) return no("invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1)");
    if (!no.have_device()) return 0;
    const cudaStream_t st = (cudaStream_t)stream;
    WsGuard guard(st);
    const long long se = nf <= 0 || len <= 0 || inc == 1 ? 0 : strided_scratch_elems(nf, len);
    T* scr = se ? (T*)ws_get(al((size_t)se * sizeof(T))) : nullptr;
    // the table's largest entry for the lane guard, and whether every entry is > 0 (the lane engine's condition): one read-back
    std::vector<T> tab(nf > 0 ? (size_t)(nf / fpi) : 0);
    if (!tab.empty() && !(no.cuda_ok(cudaMemcpyAsync(tab.data(), lamf, tab.size() * sizeof(T), cudaMemcpyDeviceToHost, st)) &&
                          no.cuda_ok(cudaStreamSynchronize(st)))) return 0;
    bool pos = true; double lmax = 0.0;
    for (T v : tab) { pos = pos && v > T(0); if ((double)v > lmax) lmax = (double)v; }
    const Engine eng = (nf >= 1024 && len >= 64) ? lane_guard<T>((Engine)g_engine, in, nf * (long long)len, lmax, st) : (Engine)g_engine;
    return no.cuda_ok(prox_fibers_lamf<T>(in, nullptr, IN_A, out, FiberGeom{nf, len, inc}, lamf, fpi, pos, eng, scr, st, se));
}

// The segmentation tape with fiber j's penalty lamf[j / fpi]; the refusals of dev_tape, then the groups (fpi >= 1, nf a multiple of fpi,
// fpi a multiple of inc: every group is whole slabs).
template <typename T>
static int dev_tape_lamf(const char* fn, const T* y, long long nf, int len, long long inc, const T* lamf, long long fpi, uint32_t* F,
                         uint32_t* U, void* stream) {
    const Refuse no{fn};
    if (nf < 0 || len < 0 || inc < 1 || nf % inc != 0) return no("invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)");
    if (!y || !F || !U || !lamf) return no("NULL array");
    if (fpi < 1 || nf % fpi != 0 || fpi % inc != 0) return no("invalid penalty groups (need fpi >= 1, nf a multiple of fpi, fpi a multiple of inc)");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    return no.cuda_ok(ptvv::fiber_tape_lamf<T>(y, nf, len, inc, lamf, fpi, F, U, (cudaStream_t)stream));
}

// Segmentation tape of y over the fibers (nf, len, inc) (nf a multiple of inc); refused calls write nothing.
template <typename T>
static int dev_tape(const char* fn, const T* y, long long nf, int len, long long inc, T lam, const T* lamv, uint32_t* F, uint32_t* U,
                    void* stream) {
    const Refuse no{fn};
    if (nf < 0 || len < 0 || inc < 1 || (nf > 0 && nf % inc != 0))
        return no("invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)");
    if (nf == 0 || len == 0) return 1;
    if (!y || !F || !U) return no("NULL array");
    if (!lamv && !(lam >= 0)) return no("negative penalty");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    return no.cuda_ok(ptvv::fiber_tape<T>(y, nf, len, inc, lam, lamv, F, U, (cudaStream_t)stream));
}

template <typename T>
static int dev_vjp_tape(const char* fn, const uint32_t* F, const uint32_t* U, const T* g, T* gx, T* gw, long long nf, int len, long long inc,
                        void* stream) {
    const Refuse no{fn};
    if (nf < 0 || len < 0 || inc < 1 || (nf > 0 && nf % inc != 0))
        return no("invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)");
    if (nf == 0 || len == 0) return 1;
    if (!F || !U || !g || !gx) return no("NULL array");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    const size_t sb = ptvv::vjp_scratch_bytes(nf, len);
    void* scr = sb ? ws_get(sb) : nullptr;
    if (sb && !scr) return no("out of device memory");
    return no.cuda_ok(ptvv::vjp_fibers_tape<T>(F, U, g, gx, gw, nf, len, inc, scr, (cudaStream_t)stream));
}

template <typename T>
static int dev_dr2_record(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, T W1, T W2, T* out, int maxit, void* tape,
                          size_t tape_bytes, double* info, void* stream) {
    const Refuse no{fn, info, 1};
    if (M < 1 || N < 1 || batch < 1) return no("invalid shape (need M, N, batch >= 1)");
    if (!Y || !out || !tape) return no("NULL array");
    if (!(W1 >= 0) || !(W2 >= 0)) return no("negative penalty");
    if (tape_bytes < dr2_tape_bytes(M, N, batch, maxit)) return no("tape_bytes smaller than proxtv_DR2_TV_tape_bytes()");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = ws_get(ws_bytes_dr2_record<T>(M, N, batch));
    if (!ws) return no("out of memory");
    if (!no.cuda_ok(dr2_record_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, tape, ws, (Engine)g_engine, (cudaStream_t)stream)))
        return 0;
    if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; }
    return 1;
}

template <typename T>
static int dev_dr2_vjp(const char* fn, size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY,
                       double* glam, void* stream) {
    const Refuse no{fn};
    if (M < 1 || N < 1 || batch < 1) return no("invalid shape (need M, N, batch >= 1)");
    if (!tape || !gout || !gY) return no("NULL array");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = dr2_tape_check(tape, sizeof(T), M, N, batch, row_major, maxit, (cudaStream_t)stream)) return no(why);
    void* ws = ws_get(ws_bytes_dr2_vjp<T>(M, N, batch));
    if (!ws) return no("out of memory");
    return no.cuda_ok(dr2_vjp_device<T>(M, N, batch, row_major, maxit, tape, gout, gY, glam, ws, (cudaStream_t)stream));
}

template <typename T>
static int dev_drw_record(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit,
                          void* tape, size_t tape_bytes, double* info, void* stream) {
    const Refuse no{fn, info, 1};
    if (M < 1 || N < 1 || batch < 1) return no("invalid shape (need M, N, batch >= 1)");
    if (!Y || !out || !tape || (M > 1 && !W1) || (N > 1 && !W2)) return no("NULL array");
    if (tape_bytes < drw_tape_bytes(M, N, batch, maxit)) return no("tape_bytes smaller than proxtv_DR2L1W_TV_batched_tape_bytes()");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = ws_get(ws_bytes_drw_record<T>(M, N, batch));
    if (!ws) return no("out of memory");
    if (!no.cuda_ok(drw_record_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, tape, ws, (Engine)g_engine, (cudaStream_t)stream)))
        return 0;
    if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; }
    return 1;
}

template <typename T>
static int dev_drw_vjp(const char* fn, size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY, T* gW1,
                       T* gW2, void* stream) {
    const Refuse no{fn};
    if (M < 1 || N < 1 || batch < 1) return no("invalid shape (need M, N, batch >= 1)");
    if (!tape || !gout || !gY) return no("NULL array");
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = drw_tape_check(tape, sizeof(T), M, N, batch, row_major, maxit, (cudaStream_t)stream)) return no(why);
    void* ws = ws_get(ws_bytes_drw_vjp<T>(M, N, batch));
    if (!ws) return no("out of memory");
    return no.cuda_ok(drw_vjp_device<T>(M, N, batch, row_major, maxit, tape, gout, gY, gW1, gW2, ws, (cudaStream_t)stream));
}

// The shape bounds of the tape paths (the header holds up to PDR_TAPE_MAX_DIMS axes): nullptr when valid, else the reason.
const char* nd_shape_check(NdSolver s, const int* ns, int nds, int npen) {
    if (s == ND_PD2 && (npen < 1 || npen > 2)) return "PD2_TV takes 1 or 2 penalty terms";
    if (nds < 1 || nds > PDR_TAPE_MAX_DIMS) return "invalid dimensions (need 1 <= nds <= 16)";
    for (int i = 0; i < nds; i++) if (ns[i] < 0) return "invalid dimensions (negative size)";
    if (npen < 1 || npen > 64) return "need 1 to 64 penalty terms";
    return nullptr;
}

// Arguments of the tape entry points: nullptr when valid (t filled), else the reason.
const char* nd_args_check(NdSolver s, const int* ns, int nds, int npen, const double* dims, NdTerms* t) {
    if (const char* why = nd_shape_check(s, ns, nds, npen)) return why;
    return nd_terms(ns, nds, npen, dims, t);
}

size_t nd_tape_bytes_checked(NdSolver s, const int* ns, int nds, int npen, int maxIters) {
    return !ns || nd_shape_check(s, ns, nds, npen) ? 0 : nd_tape_bytes(s, ns, nds, npen, maxIters);
}

// The solver s as proxtv_<solver>_dev_* computes it (the same device solver call), writing the tape and, after the solve, its header;
// every refusal comes before anything is written, lambdas included.
template <typename T>
static int dev_nd_record(const char* fn, NdSolver s, const T* y, double* lambdas, const double* dims, T* x, double* info, const int* ns,
                         int nds, int npen, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    static const char* const too_small[3] = {"tape_bytes smaller than proxtv_PD2_TV_tape_bytes()",
                                             "tape_bytes smaller than proxtv_PD_TV_tape_bytes()",
                                             "tape_bytes smaller than proxtv_PDR_TV_tape_bytes()"};
    const Refuse no{fn, info, 1};
    if (!y || !x || !lambdas || !dims || !ns || !tape) return no("NULL array");
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) return no(why);
    for (int i = 0; i < npen; i++) if (!(lambdas[i] >= 0)) return no("negative penalty");
    const size_t need = nd_tape_bytes(s, ns, nds, npen, maxIters);
    if (need == 0) return no("tape size does not fit in size_t (maxIters too large)");
    if (tape_bytes < need) return no(too_small[s]);
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = ws_get(ws_bytes_pd<T>(t.n, npen));
    if (!ws) return no("out of memory");
    double linfo[3] = {0, 0, RC_OK};                   // the header needs the iteration count even when the caller passes no info
    double* pinfo = info ? info : linfo;
    scale_penalties(s, lambdas, npen);
    if (!nd_solve<T>(s, y, lambdas, dims, x, pinfo, ns, nds, npen, maxIters, ws, (cudaStream_t)stream, tape)) return no("device solver failed");
    return no.cuda_ok(nd_tape_header(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, (int)pinfo[INFO_ITERS], (cudaStream_t)stream));
}

template <typename T>
static int dev_nd_vjp(const char* fn, NdSolver s, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters,
                      const void* tape, const T* gout, T* gY, double* glam, void* stream) {
    const Refuse no{fn};
    if (!ns || !dims || !tape || !gout || !gY) return no("NULL array");
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) return no(why);
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = nd_tape_check(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, iters, (cudaStream_t)stream)) return no(why);
    void* ws = ws_get(ws_bytes_nd_vjp<T>(t, npen, glam != nullptr));
    if (!ws) return no("out of memory");
    return no.cuda_ok(nd_vjp_device<T>(s, t, npen, maxIters, iters, tape, gout, gY, glam, ws, (cudaStream_t)stream));
}

// ---- batched PD_TV / PD2_TV (DESIGN.md section 16): `batch` items of prod(ns) elements back to back, each with its own stop rule ----
// Every refusal writes info[3 b + RC] = RC_ERROR for every item and nothing else; lambdas are never written (PD_TV's factor npen is
// applied to a copy).  items: lambdas holds one row of npen penalties per item, item-major (section 16.1), else one row for all.

// The solve (host_io: y and x are host arrays) or, given a tape, the recorded solve and then the tape's header and K table.
template <typename T>
static int run_pd_batched(const char* fn, NdSolver s, bool host_io, bool record, const T* y, const double* lambdas, const double* dims, T* x, double* info,
                          const int* ns, int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, cudaStream_t st,
                          bool items = false) {
    static const char* const too_small[2] = {"tape_bytes smaller than proxtv_PD2_TV_batched_tape_bytes()",
                                             "tape_bytes smaller than proxtv_PD_TV_batched_tape_bytes()"};
    const Refuse no{fn, info, batch};
    NdTerms t;
    if (record) {                                      // the order of the single-item record entry points
        if (!y || !x || !lambdas || !dims || !ns || !tape) return no("NULL array");
        if (batch < 1) return no("invalid batch (need batch >= 1)");
        if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) return no(why);
        for (long long i = 0; i < (long long)npen * (items ? batch : 1); i++) if (!(lambdas[i] >= 0)) return no("negative penalty");
        const size_t need = nd_tape_bytes(s, ns, nds, npen, maxIters, batch);
        if (need == 0) return no("tape size does not fit in size_t (maxIters too large)");
        if (tape_bytes < need) return no(too_small[s]);
        if (!no.have_device()) return 0;
    } else {                                           // the order of the single-item solve entry points
        if (!no.have_device()) return 0;
        if (nds <= 0 || !ns) return no("invalid dimensions");
        if (batch < 1) return no("invalid batch (need batch >= 1)");
        if (!y || !x || (npen > 0 && (!lambdas || !dims))) return no("NULL array");
        if (s == ND_PD2 && npen > 2) return no("this algorithm can not work with more than 2 penalties");
        if (s == ND_PD2 && npen < 1) return no("invalid penalty dimensions");
        if (const char* why = nd_terms(ns, nds, npen, dims, &t)) return no(why);
        if (items && !lambdas) return no("NULL array");
    }
    const long long n = t.n;
    WsGuard guard(st);
    const int rows = items ? batch : 1;
    std::vector<double> lam(lambdas ? lambdas : nullptr, lambdas ? lambdas + (npen > 0 ? (size_t)npen * rows : 0) : nullptr);
    for (int b = 0; b < rows && npen > 0; b++) scale_penalties(s, lam.data() + (size_t)b * npen, npen);
    const int lstride = items ? npen : 0;
    void* ws = ws_get(ws_bytes_pd<T>(n, npen, batch));
    if (!ws) return no("out of memory");
    std::vector<double> linfo(3 * (size_t)batch);      // the tape's K table needs the rows even when the caller passes no info
    double* pinfo = info ? info : linfo.data();
    const size_t nt = (size_t)n * batch;
    HostIO<T> io(no, st);
    if (host_io && nt > 0) {
        io.in(y, nt); io.out(x, nt);
        if (!io.stage()) return 0;
    }
    const int ok = s == ND_PD2 ? pd2_device<T>(y, lam.data(), dims, x, pinfo, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape, batch, lstride)
                               : pd_device<T>(y, lam.data(), dims, x, pinfo, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape, batch, lstride);
    if (!ok) return no("device solver failed");
    if (record && !no.cuda_ok(nd_tape_header_batched(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, batch, pinfo, st))) return 0;
    return io.finish() ? 1 : 0;
}

template <typename T>
static int dev_nd_vjp_batched(const char* fn, NdSolver s, const int* ns, int nds, int npen, const double* dims, int batch, int maxIters,
                              const void* tape, const T* gout, T* gY, double* glam, void* stream) {
    const Refuse no{fn};
    if (!ns || !dims || !tape || !gout || !gY) return no("NULL array");
    if (batch < 1) return no("invalid batch (need batch >= 1)");
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) return no(why);
    if (!no.have_device()) return 0;
    WsGuard guard((cudaStream_t)stream);
    std::vector<int> K(batch);
    if (const char* why = nd_tape_check_batched(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, batch, K.data(), (cudaStream_t)stream))
        return no(why);
    void* ws = ws_get(ws_bytes_nd_vjp<T>(t, npen, glam != nullptr, batch));
    if (!ws) return no("out of memory");
    return no.cuda_ok(nd_vjp_device<T>(s, t, npen, maxIters, 0, tape, gout, gY, glam, ws, (cudaStream_t)stream, batch, K.data()));
}

// The lane engine's hooks for the tools: no stdout line, and proxtv_last_error() only for a CUDA error.
template <typename T>
int lane_hook(const char* fn, int op, const T* A, const T* B, const T* C, T* X, T* X2, long long nf, int len, long long inc, T lam, void* stream) {
    WsGuard guard((cudaStream_t)stream);
    void* scr = ptvl::lane_scratch(nf, len);
    if (!scr) return 0;
    const cudaError_t e = ptvl::lane_prox<T>(op, A, B, C, X, nf, len, inc, lam, scr, (cudaStream_t)stream, X2);
    if (e != cudaSuccess) { cudaGetLastError(); Refuse{fn}.note(cudaGetErrorString(e)); return 0; }
    return 1;
}

size_t nd_tape_bytes_batched(NdSolver s, const int* ns, int nds, int npen, int batch, int maxIters) {
    return !ns || batch < 1 || nd_shape_check(s, ns, nds, npen) ? 0 : nd_tape_bytes(s, ns, nds, npen, maxIters, batch);
}

}  // namespace

extern "C" {

int proxtv_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }
const char* proxtv_last_error(void) { return g_err.c_str(); }
const char* proxtv_version(void) { return "proxtv_b200 0.1 (sm_90a)"; }
int proxtv_set_engine(int e) { int o = g_engine; if (e >= 0 && e <= 8) g_engine = e; return o; }
void* proxtv_host_alloc(size_t bytes) { void* p = nullptr; if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
void proxtv_host_free(void* p) { if (p) cudaFreeHost(p); }
void proxtv_profile_enable(int on) { profile_enable(on); }
void proxtv_profile_reset(void) { profile_reset(); }
void proxtv_profile_read(double* ms, long long* launches, long long* spans) { profile_read(ms, launches, spans); }
void proxtv_release_workspace(void) { std::lock_guard<std::recursive_mutex> lk(g_mu); for (int d = 0; d < MAX_DEVICES; d++) { g_ws_d[d].release(); g_io_d[d].release(); } }

// ---- experimental: the lane-per-fiber streaming engine (kernels_lane.cu), device pointers ----
int proxtv_lane_prox_dev_f64(int op, const double* A, const double* B, const double* C, double* X, long long nf, int len, long long inc,
                             double lam, void* stream) {
    return lane_hook<double>("proxtv_lane_prox_dev_f64", op, A, B, C, X, nullptr, nf, len, inc, lam, stream);
}
int proxtv_lane_prox2_dev_f64(int op, const double* A, const double* B, const double* C, double* X, double* X2, long long nf, int len, long long inc,
                              double lam, void* stream) {
    return lane_hook<double>("proxtv_lane_prox2_dev_f64", op, A, B, C, X, X2, nf, len, inc, lam, stream);
}
int proxtv_lane_prox_dev_f32(int op, const float* A, const float* B, const float* C, float* X, long long nf, int len, long long inc,
                             float lam, void* stream) {
    return lane_hook<float>("proxtv_lane_prox_dev_f32", op, A, B, C, X, nullptr, nf, len, inc, lam, stream);
}
void proxtv_lane_tuning(int clen, int halo, int variant) { ptvl::lane_set_tuning(clen, halo, variant); }
void proxtv_lane_tasklog(unsigned long long* dev, long long cap_tasks) { ptvl::lane_set_tasklog(dev, cap_tasks); }
int proxtv_lane_guard_last(void) { return lane_guard_last(); }
int proxtv_long_fiber_last(void) { return long_fiber_last(); }
unsigned long long proxtv_lane_stats(int reset) { return ptvl::lane_read_stats(reset); }

// ---- Part 1: drop-in symbols ----
void hybridTautString_TV1(double* y, int n, double lambda, double* x) {
    run_prox_fibers<double>("hybridTautString_TV1", true, y, x, 1, n, 1, lambda, nullptr, 0);
}
void hybridTautString_TV1_custom(double* y, int n, double lambda, double* x, double) {
    run_prox_fibers<double>("hybridTautString_TV1_custom", true, y, x, 1, n, 1, lambda, nullptr, 0);
}
int classicTautString_TV1(double* signal, int n, double lam, double* prox) {
    if (n <= 0) return 1;
    if (lam <= 0 || n == 1) { memmove(prox, signal, (size_t)n * sizeof(double)); return 1; }   // TVL1opt_tautstring.cpp:258-263
    run_prox_fibers<double>("classicTautString_TV1", true, signal, prox, 1, n, 1, lam, nullptr, 0);
    return 1;
}
int linearizedTautString_TV1(double* y, double lambda, double* x, int n) {
    run_prox_fibers<double>("linearizedTautString_TV1", true, y, x, 1, n, 1, lambda, nullptr, 0);
    return 1;
}
void TV1D_denoise(double* input, double* output, const int width, const double lambda) {
    if (width > 0 && lambda >= 0) run_prox_fibers<double>("TV1D_denoise", true, input, output, 1, width, 1, lambda, nullptr, 0);
}
int tautString_TV1_Weighted(double* y, double* lambda, double* x, int n) {
    if (n == 1) { x[0] = y[0]; return 1; }
    run_prox_fibers<double>("tautString_TV1_Weighted", true, y, x, 1, n, 1, 0.0, lambda, 0);
    return 1;
}
// The reference's alternative 1D TV-L1 solvers compute the same unique minimiser (<= 4e-14 apart on random data, 9e-7 for Condat's
// float-truncating taut-string variant -- measured with the compiled reference): they all map onto the exact kernel.
static void ok_info(double* info) { if (info) { info[INFO_ITERS] = 0; info[INFO_GAP] = 0; info[INFO_RC] = RC_OK; } }
int PN_TV1(double* y, double lambda, double* x, double* info, int n, double, void*) {
    if (!run_prox_fibers<double>("PN_TV1", true, y, x, 1, n, 1, lambda, nullptr, 0)) return Refuse{"PN_TV1", info, 1}.mark();
    ok_info(info); return 1;
}
int PN_TV1_Weighted(double* Y, double* W, double* X, double* info, int n, double, void*) {
    if (n == 1) { X[0] = Y[0]; ok_info(info); return 1; }
    if (!run_prox_fibers<double>("PN_TV1_Weighted", true, Y, X, 1, n, 1, 0.0, W, 0)) return Refuse{"PN_TV1_Weighted", info, 1}.mark();
    ok_info(info); return 1;
}
void TV1D_denoise_tautstring(double* input, double* output, int width, const double lambda) {
    if (width > 0 && lambda >= 0) run_prox_fibers<double>("TV1D_denoise_tautstring", true, input, output, 1, width, 1, lambda, nullptr, 0);
}
void SolveTVConvexQuadratic_a1_nw(int n, double* b, double w, double* solution) {
    run_prox_fibers<double>("SolveTVConvexQuadratic_a1_nw", true, b, solution, 1, n, 1, w, nullptr, 0);
}
void SolveTVConvexQuadratic_a1(int n, double* b, double* w, double* solution) {
    if (n == 1) { solution[0] = b[0]; return; }
    run_prox_fibers<double>("SolveTVConvexQuadratic_a1", true, b, solution, 1, n, 1, 0.0, w, 0);
}
void dp(int n, double* y, double lam, double* beta) {
    run_prox_fibers<double>("dp", true, y, beta, 1, n, 1, lam, nullptr, 0);
}
int TV(double* y, double lambda, double* x, double* info, int n, double p, void*) {
    const Refuse no{"TVopt", info, 1};
    if (p < 1) return no("TV only works for norms p >= 1");                                         // TVgenopt.cpp:37-38
    if (p != 1) return no("only p = 1 (TV-L1) is implemented on the GPU path");
    if (!run_prox_fibers<double>("TVopt", true, y, x, 1, n, 1, lambda, nullptr, 0)) return no.mark();
    if (info) { info[INFO_RC] = RC_OK; info[INFO_ITERS] = 0; info[INFO_GAP] = 0; }                 // :43-47
    return 1;
}
int DR2_TV(size_t M, size_t N, double* unary, double W1, double W2, double norm1, double norm2, double* s, int, int maxit,
           double* info) {
    if (norm1 != 1.0 || norm2 != 1.0) return Refuse{"DR2_TV", info, 1}("only p = 1 (TV-L1) penalties are implemented on the GPU path");
    return run_dr2<double>("DR2_TV", true, M, N, 1, 0, unary, W1, W2, s, maxit, info, 0);
}
int DR2L1W_TV(size_t M, size_t N, double* unary, double* W1, double* W2, double* s, int, int maxit, double* info) {
    return run_drw<double>("DR2L1W_TV", true, M, N, 1, 0, unary, W1, W2, s, maxit, info, 0);
}
int CondatChambollePock2_TV(size_t M, size_t N, double* Y, double lambda, double* X, short alg, int maxit, double* info) {
    return run_cp2<double>("Condat2_TV", true, M, N, 1, 0, Y, lambda, false, nullptr, nullptr, X, alg, maxit, info, 0);
}
int PD2_TV(double* y, double* lambdas, double* norms, double* dims, double* x, double* info, int* ns, int nds, int npen, int,
           int maxIters) {
    return run_pd<double>("PD2_TV", ND_PD2, true, y, lambdas, norms, dims, x, info, ns, nds, npen, maxIters, 0);
}
int PD_TV(double* y, double* lambdas, double* norms, double* dims, double* x, double* info, int* ns, int nds, int npen, int,
          int maxIters) {
    return run_pd<double>("PD_TV", ND_PD, true, y, lambdas, norms, dims, x, info, ns, nds, npen, maxIters, 0);
}
int PDR_TV(double* y, double* lambdas, double* norms, double* dims, double* x, double* info, int* ns, int nds, int npen, int,
           int maxIters) {
    return run_pd<double>("PDR_TV", ND_PDR, true, y, lambdas, norms, dims, x, info, ns, nds, npen, maxIters, 0);
}

// ---- Part 2: extensions ----
int proxtv_prox_fibers_dev_f64(const double* in, double* out, long long nf, int len, long long inc, double lam, const double* lamv, void* stream) {
    return run_prox_fibers<double>("proxtv_prox_fibers_dev_f64", false, in, out, nf, len, inc, lam, lamv, (cudaStream_t)stream);
}
int proxtv_prox_fibers_dev_f32(const float* in, float* out, long long nf, int len, long long inc, float lam, const float* lamv, void* stream) {
    return run_prox_fibers<float>("proxtv_prox_fibers_dev_f32", false, in, out, nf, len, inc, lam, lamv, (cudaStream_t)stream);
}
int proxtv_prox_fibers_vjp_dev_f64(const double* y, const double* g, double* gx, double* gw, long long nf, int len, long long inc, double lam,
                                   const double* lamv, void* stream) {
    return dev_vjp<double>("proxtv_prox_fibers_vjp_dev_f64", y, g, gx, gw, nf, len, inc, lam, lamv, stream);
}
int proxtv_prox_fibers_vjp_dev_f32(const float* y, const float* g, float* gx, float* gw, long long nf, int len, long long inc, float lam,
                                   const float* lamv, void* stream) {
    return dev_vjp<float>("proxtv_prox_fibers_vjp_dev_f32", y, g, gx, gw, nf, len, inc, lam, lamv, stream);
}
void proxtv_vjp_tuning(int chunk_len) { ptvv::vjp_set_tuning(chunk_len); }
int proxtv_fiber_tape_dev_f64(const double* y, long long nf, int len, long long inc, double lam, const double* lamv, unsigned* F, unsigned* U,
                              void* stream) {
    return dev_tape<double>("proxtv_fiber_tape_dev_f64", y, nf, len, inc, lam, lamv, F, U, stream);
}
int proxtv_fiber_tape_dev_f32(const float* y, long long nf, int len, long long inc, float lam, const float* lamv, unsigned* F, unsigned* U,
                              void* stream) {
    return dev_tape<float>("proxtv_fiber_tape_dev_f32", y, nf, len, inc, lam, lamv, F, U, stream);
}
int proxtv_prox_fibers_vjp_tape_dev_f64(const unsigned* F, const unsigned* U, const double* g, double* gx, double* gw, long long nf, int len,
                                        long long inc, void* stream) {
    return dev_vjp_tape<double>("proxtv_prox_fibers_vjp_tape_dev_f64", F, U, g, gx, gw, nf, len, inc, stream);
}
int proxtv_prox_fibers_vjp_tape_dev_f32(const unsigned* F, const unsigned* U, const float* g, float* gx, float* gw, long long nf, int len,
                                        long long inc, void* stream) {
    return dev_vjp_tape<float>("proxtv_prox_fibers_vjp_tape_dev_f32", F, U, g, gx, gw, nf, len, inc, stream);
}
int proxtv_prox_fibers_f64(const double* in, double* out, long long nf, int len, long long inc, double lam, const double* lamv) {
    return run_prox_fibers<double>("proxtv_prox_fibers_f64", true, in, out, nf, len, inc, lam, lamv, 0);
}
int proxtv_prox_fibers_f32(const float* in, float* out, long long nf, int len, long long inc, float lam, const float* lamv) {
    return run_prox_fibers<float>("proxtv_prox_fibers_f32", true, in, out, nf, len, inc, lam, lamv, 0);
}

int proxtv_DR2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double W1, double W2, double* out, int maxit, double* info, void* stream) {
    return run_dr2<double>("proxtv_DR2_TV_dev_f64", false, M, N, batch, row_major, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
int proxtv_DR2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, float W1, float W2, float* out, int maxit, double* info, void* stream) {
    return run_dr2<float>("proxtv_DR2_TV_dev_f32", false, M, N, batch, row_major, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
size_t proxtv_DR2_TV_tape_bytes(size_t M, size_t N, int batch, int maxit) { return batch < 1 ? 0 : dr2_tape_bytes(M, N, batch, maxit); }
int proxtv_DR2_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double W1, double W2, double* out, int maxit,
                                 void* tape, size_t tape_bytes, double* info, void* stream) {
    return dev_dr2_record<double>("proxtv_DR2_TV_record_dev_f64", M, N, batch, row_major, Y, W1, W2, out, maxit, tape, tape_bytes, info, stream); }
int proxtv_DR2_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, float W1, float W2, float* out, int maxit,
                                 void* tape, size_t tape_bytes, double* info, void* stream) {
    return dev_dr2_record<float>("proxtv_DR2_TV_record_dev_f32", M, N, batch, row_major, Y, W1, W2, out, maxit, tape, tape_bytes, info, stream); }
int proxtv_DR2_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const double* gout, double* gY,
                              double* glam, void* stream) {
    return dev_dr2_vjp<double>("proxtv_DR2_TV_vjp_dev_f64", M, N, batch, row_major, maxit, tape, gout, gY, glam, stream); }
int proxtv_DR2_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const float* gout, float* gY,
                              double* glam, void* stream) {
    return dev_dr2_vjp<float>("proxtv_DR2_TV_vjp_dev_f32", M, N, batch, row_major, maxit, tape, gout, gY, glam, stream); }
int proxtv_DR2_TV_batched_f64(size_t M, size_t N, int batch, const double* Y, double W1, double W2, double* out, int maxit, double* info) {
    return run_dr2<double>("proxtv_DR2_TV_batched_f64", true, M, N, batch, 0, Y, W1, W2, out, maxit, info, 0); }
int proxtv_DR2_TV_batched_f32(size_t M, size_t N, int batch, const float* Y, float W1, float W2, float* out, int maxit, double* info) {
    return run_dr2<float>("proxtv_DR2_TV_batched_f32", true, M, N, batch, 0, Y, W1, W2, out, maxit, info, 0); }

int proxtv_CP2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double lambda, double* X, int alg, int maxit,
                          double* info, void* stream) {
    return run_cp2<double>("proxtv_CP2_TV_dev_f64", false, M, N, batch, row_major, Y, lambda, false, nullptr, nullptr,
                           X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, double lambda, float* X, int alg, int maxit,
                          double* info, void* stream) {
    return run_cp2<float>("proxtv_CP2_TV_dev_f32", false, M, N, batch, row_major, Y, lambda, false, nullptr, nullptr,
                           X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double lambda, double* X, int alg, int maxit,
                              double* info) {
    return run_cp2<double>("proxtv_CP2_TV_batched_f64", true, M, N, batch, row_major, Y, lambda, false, nullptr, nullptr, X, alg, maxit, info, 0); }
int proxtv_CP2_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float* Y, double lambda, float* X, int alg, int maxit,
                              double* info) {
    return run_cp2<float>("proxtv_CP2_TV_batched_f32", true, M, N, batch, row_major, Y, lambda, false, nullptr, nullptr, X, alg, maxit, info, 0); }

int proxtv_CP2W_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2, double* X,
                           int alg, int maxit, double* info, void* stream) {
    return run_cp2<double>("proxtv_CP2W_TV_dev_f64", false, M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2W_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2, float* X,
                           int alg, int maxit, double* info, void* stream) {
    return run_cp2<float>("proxtv_CP2W_TV_dev_f32", false, M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2W_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2,
                               double* X, int alg, int maxit, double* info) {
    return run_cp2<double>("proxtv_CP2W_TV_batched_f64", true, M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, 0); }
int proxtv_CP2W_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2, float* X,
                               int alg, int maxit, double* info) {
    return run_cp2<float>("proxtv_CP2W_TV_batched_f32", true, M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, 0); }

size_t proxtv_CP2_TV_tape_bytes(size_t M, size_t N, int batch) { return batch < 1 ? 0 : cp2_tape_bytes(M, N, batch); }
int proxtv_CP2_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double lambda, double* X, int alg, int maxit,
                                 double* info, void* tape, size_t tape_bytes, void* stream) {
    return dev_cp2_record<double>("proxtv_CP2_TV_record_dev_f64", M, N, batch, row_major, Y, lambda, false, nullptr, nullptr, X, alg, maxit, info,
                                  tape, tape_bytes, stream); }
int proxtv_CP2_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, double lambda, float* X, int alg, int maxit,
                                 double* info, void* tape, size_t tape_bytes, void* stream) {
    return dev_cp2_record<float>("proxtv_CP2_TV_record_dev_f32", M, N, batch, row_major, Y, lambda, false, nullptr, nullptr, X, alg, maxit, info,
                                 tape, tape_bytes, stream); }
int proxtv_CP2W_TV_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2, double* X,
                                  int alg, int maxit, double* info, void* tape, size_t tape_bytes, void* stream) {
    return dev_cp2_record<double>("proxtv_CP2W_TV_record_dev_f64", M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, tape,
                                  tape_bytes, stream); }
int proxtv_CP2W_TV_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2, float* X,
                                  int alg, int maxit, double* info, void* tape, size_t tape_bytes, void* stream) {
    return dev_cp2_record<float>("proxtv_CP2W_TV_record_dev_f32", M, N, batch, row_major, Y, 0., true, W1, W2, X, alg, maxit, info, tape,
                                 tape_bytes, stream); }
int proxtv_CP2_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, const void* tape, const double* X, const double* gout, double* gY,
                              double* glam, void* stream) {
    return dev_cp2_vjp<double>("proxtv_CP2_TV_vjp_dev_f64", false, M, N, batch, row_major, tape, X, gout, gY, nullptr, nullptr, glam, stream); }
int proxtv_CP2_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, const void* tape, const float* X, const float* gout, float* gY,
                              double* glam, void* stream) {
    return dev_cp2_vjp<float>("proxtv_CP2_TV_vjp_dev_f32", false, M, N, batch, row_major, tape, X, gout, gY, nullptr, nullptr, glam, stream); }
int proxtv_CP2W_TV_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, const void* tape, const double* X, const double* gout, double* gY,
                               double* gW1, double* gW2, double* glam, void* stream) {
    return dev_cp2_vjp<double>("proxtv_CP2W_TV_vjp_dev_f64", true, M, N, batch, row_major, tape, X, gout, gY, gW1, gW2, glam, stream); }
int proxtv_CP2W_TV_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, const void* tape, const float* X, const float* gout, float* gY,
                               float* gW1, float* gW2, double* glam, void* stream) {
    return dev_cp2_vjp<float>("proxtv_CP2W_TV_vjp_dev_f32", true, M, N, batch, row_major, tape, X, gout, gY, gW1, gW2, glam, stream); }

int proxtv_DR2L1W_TV_dev_f64(size_t M, size_t N, const double* Y, const double* W1, const double* W2, double* out, int maxit, double* info, void* stream) {
    return run_drw<double>("proxtv_DR2L1W_TV_dev_f64", false, M, N, 1, 0, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
int proxtv_DR2L1W_TV_dev_f32(size_t M, size_t N, const float* Y, const float* W1, const float* W2, float* out, int maxit, double* info, void* stream) {
    return run_drw<float>("proxtv_DR2L1W_TV_dev_f32", false, M, N, 1, 0, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
size_t proxtv_DR2L1W_TV_tape_bytes(size_t M, size_t N, int maxit) { return drw_tape_bytes(M, N, 1, maxit); }
int proxtv_DR2L1W_TV_record_dev_f64(size_t M, size_t N, const double* Y, const double* W1, const double* W2, double* out, int maxit, void* tape,
                                    size_t tape_bytes, double* info, void* stream) {
    return dev_drw_record<double>("proxtv_DR2L1W_TV_record_dev_f64", M, N, 1, 0, Y, W1, W2, out, maxit, tape, tape_bytes, info, stream); }
int proxtv_DR2L1W_TV_record_dev_f32(size_t M, size_t N, const float* Y, const float* W1, const float* W2, float* out, int maxit, void* tape,
                                    size_t tape_bytes, double* info, void* stream) {
    return dev_drw_record<float>("proxtv_DR2L1W_TV_record_dev_f32", M, N, 1, 0, Y, W1, W2, out, maxit, tape, tape_bytes, info, stream); }
int proxtv_DR2L1W_TV_vjp_dev_f64(size_t M, size_t N, int maxit, const void* tape, const double* gout, double* gY, double* gW1, double* gW2,
                                 void* stream) {
    return dev_drw_vjp<double>("proxtv_DR2L1W_TV_vjp_dev_f64", M, N, 1, 0, maxit, tape, gout, gY, gW1, gW2, stream); }
int proxtv_DR2L1W_TV_vjp_dev_f32(size_t M, size_t N, int maxit, const void* tape, const float* gout, float* gY, float* gW1, float* gW2,
                                 void* stream) {
    return dev_drw_vjp<float>("proxtv_DR2L1W_TV_vjp_dev_f32", M, N, 1, 0, maxit, tape, gout, gY, gW1, gW2, stream); }
size_t proxtv_DR2L1W_TV_batched_tape_bytes(size_t M, size_t N, int batch, int maxit) { return batch < 1 ? 0 : drw_tape_bytes(M, N, batch, maxit); }
int proxtv_DR2L1W_TV_batched_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2, double* out,
                                     int maxit, double* info, void* stream) {
    return run_drw<double>("proxtv_DR2L1W_TV_batched_dev_f64", false, M, N, batch, row_major, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
int proxtv_DR2L1W_TV_batched_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2, float* out,
                                     int maxit, double* info, void* stream) {
    return run_drw<float>("proxtv_DR2L1W_TV_batched_dev_f32", false, M, N, batch, row_major, Y, W1, W2, out, maxit, info, (cudaStream_t)stream); }
int proxtv_DR2L1W_TV_batched_record_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2,
                                            double* out, int maxit, void* tape, size_t tape_bytes, double* info, void* stream) {
    return dev_drw_record<double>("proxtv_DR2L1W_TV_batched_record_dev_f64", M, N, batch, row_major, Y, W1, W2, out, maxit, tape, tape_bytes, info,
                                  stream); }
int proxtv_DR2L1W_TV_batched_record_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2,
                                            float* out, int maxit, void* tape, size_t tape_bytes, double* info, void* stream) {
    return dev_drw_record<float>("proxtv_DR2L1W_TV_batched_record_dev_f32", M, N, batch, row_major, Y, W1, W2, out, maxit, tape, tape_bytes, info,
                                 stream); }
int proxtv_DR2L1W_TV_batched_vjp_dev_f64(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const double* gout, double* gY,
                                         double* gW1, double* gW2, void* stream) {
    return dev_drw_vjp<double>("proxtv_DR2L1W_TV_batched_vjp_dev_f64", M, N, batch, row_major, maxit, tape, gout, gY, gW1, gW2, stream); }
int proxtv_DR2L1W_TV_batched_vjp_dev_f32(size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const float* gout, float* gY,
                                         float* gW1, float* gW2, void* stream) {
    return dev_drw_vjp<float>("proxtv_DR2L1W_TV_batched_vjp_dev_f32", M, N, batch, row_major, maxit, tape, gout, gY, gW1, gW2, stream); }
int proxtv_DR2L1W_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double* Y, const double* W1, const double* W2, double* out,
                                 int maxit, double* info) {
    return run_drw<double>("proxtv_DR2L1W_TV_batched_f64", true, M, N, batch, row_major, Y, W1, W2, out, maxit, info, 0); }
int proxtv_DR2L1W_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float* Y, const float* W1, const float* W2, float* out,
                                 int maxit, double* info) {
    return run_drw<float>("proxtv_DR2L1W_TV_batched_f32", true, M, N, batch, row_major, Y, W1, W2, out, maxit, info, 0); }

int proxtv_PD2_TV_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<double>("proxtv_PD2_TV_dev_f64", ND_PD2, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
int proxtv_PD2_TV_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<float>("proxtv_PD2_TV_dev_f32", ND_PD2, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
int proxtv_PD_TV_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<double>("proxtv_PD_TV_dev_f64", ND_PD, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
int proxtv_PD_TV_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<float>("proxtv_PD_TV_dev_f32", ND_PD, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
int proxtv_PDR_TV_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<double>("proxtv_PDR_TV_dev_f64", ND_PDR, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
int proxtv_PDR_TV_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen, int maxIters, void* stream) {
    return run_pd<float>("proxtv_PDR_TV_dev_f32", ND_PDR, false, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, (cudaStream_t)stream); }
size_t proxtv_PDR_TV_tape_bytes(const int* ns, int nds, int npen, int maxIters) { return nd_tape_bytes_checked(ND_PDR, ns, nds, npen, maxIters); }
int proxtv_PDR_TV_record_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen,
                                 int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<double>("proxtv_PDR_TV_record_dev_f64", ND_PDR, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PDR_TV_record_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen,
                                 int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<float>("proxtv_PDR_TV_record_dev_f32", ND_PDR, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PDR_TV_vjp_dev_f64(const int* ns, int nds, int npen, const double* dims, int maxIters, const void* tape, const double* gout,
                              double* gY, double* glam, void* stream) {
    return dev_nd_vjp<double>("proxtv_PDR_TV_vjp_dev_f64", ND_PDR, ns, nds, npen, dims, maxIters, 0, tape, gout, gY, glam, stream); }
int proxtv_PDR_TV_vjp_dev_f32(const int* ns, int nds, int npen, const double* dims, int maxIters, const void* tape, const float* gout,
                              float* gY, double* glam, void* stream) {
    return dev_nd_vjp<float>("proxtv_PDR_TV_vjp_dev_f32", ND_PDR, ns, nds, npen, dims, maxIters, 0, tape, gout, gY, glam, stream); }
size_t proxtv_PD_TV_tape_bytes(const int* ns, int nds, int npen, int maxIters) { return nd_tape_bytes_checked(ND_PD, ns, nds, npen, maxIters); }
size_t proxtv_PD2_TV_tape_bytes(const int* ns, int nds, int npen, int maxIters) { return nd_tape_bytes_checked(ND_PD2, ns, nds, npen, maxIters); }
int proxtv_PD_TV_record_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen,
                                int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<double>("proxtv_PD_TV_record_dev_f64", ND_PD, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PD_TV_record_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen,
                                int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<float>("proxtv_PD_TV_record_dev_f32", ND_PD, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PD2_TV_record_dev_f64(const double* y, double* lambdas, double* dims, double* x, double* info, int* ns, int nds, int npen,
                                 int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<double>("proxtv_PD2_TV_record_dev_f64", ND_PD2, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PD2_TV_record_dev_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen,
                                 int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return dev_nd_record<float>("proxtv_PD2_TV_record_dev_f32", ND_PD2, y, lambdas, dims, x, info, ns, nds, npen, maxIters, tape, tape_bytes, stream); }
int proxtv_PD_TV_vjp_dev_f64(const int* ns, int nds, int npen, const double* dims, int maxIters, int iters, const void* tape,
                             const double* gout, double* gY, double* glam, void* stream) {
    return dev_nd_vjp<double>("proxtv_PD_TV_vjp_dev_f64", ND_PD, ns, nds, npen, dims, maxIters, iters, tape, gout, gY, glam, stream); }
int proxtv_PD_TV_vjp_dev_f32(const int* ns, int nds, int npen, const double* dims, int maxIters, int iters, const void* tape,
                             const float* gout, float* gY, double* glam, void* stream) {
    return dev_nd_vjp<float>("proxtv_PD_TV_vjp_dev_f32", ND_PD, ns, nds, npen, dims, maxIters, iters, tape, gout, gY, glam, stream); }
int proxtv_PD2_TV_vjp_dev_f64(const int* ns, int nds, int npen, const double* dims, int maxIters, int iters, const void* tape,
                              const double* gout, double* gY, double* glam, void* stream) {
    return dev_nd_vjp<double>("proxtv_PD2_TV_vjp_dev_f64", ND_PD2, ns, nds, npen, dims, maxIters, iters, tape, gout, gY, glam, stream); }
int proxtv_PD2_TV_vjp_dev_f32(const int* ns, int nds, int npen, const double* dims, int maxIters, int iters, const void* tape,
                              const float* gout, float* gY, double* glam, void* stream) {
    return dev_nd_vjp<float>("proxtv_PD2_TV_vjp_dev_f32", ND_PD2, ns, nds, npen, dims, maxIters, iters, tape, gout, gY, glam, stream); }
int proxtv_PD_TV_f32(const float* y, double* lambdas, double* dims, float* x, double* info, int* ns, int nds, int npen, int maxIters) {
    return run_pd<float>("proxtv_PD_TV_f32", ND_PD, true, y, lambdas, nullptr, dims, x, info, ns, nds, npen, maxIters, 0); }

int proxtv_PD_TV_batched_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_dev_f64", ND_PD, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0,
                                (cudaStream_t)stream); }
int proxtv_PD_TV_batched_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds, int npen,
                             int batch, int maxIters) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_f64", ND_PD, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0, 0); }
int proxtv_PD_TV_batched_record_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                        int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_record_dev_f64", ND_PD, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                tape, tape_bytes, (cudaStream_t)stream); }
int proxtv_PD_TV_batched_vjp_dev_f64(const int* ns, int nds, int npen, const double* dims, int batch, int maxIters, const void* tape,
                                     const double* gout, double* gY, double* glam, void* stream) {
    return dev_nd_vjp_batched<double>("proxtv_PD_TV_batched_vjp_dev_f64", ND_PD, ns, nds, npen, dims, batch, maxIters, tape, gout, gY, glam, stream); }
int proxtv_PD_TV_batched_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_dev_f32", ND_PD, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0,
                                (cudaStream_t)stream); }
int proxtv_PD_TV_batched_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds, int npen,
                             int batch, int maxIters) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_f32", ND_PD, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0, 0); }
int proxtv_PD_TV_batched_record_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                        int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_record_dev_f32", ND_PD, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                tape, tape_bytes, (cudaStream_t)stream); }
int proxtv_PD_TV_batched_vjp_dev_f32(const int* ns, int nds, int npen, const double* dims, int batch, int maxIters, const void* tape,
                                     const float* gout, float* gY, double* glam, void* stream) {
    return dev_nd_vjp_batched<float>("proxtv_PD_TV_batched_vjp_dev_f32", ND_PD, ns, nds, npen, dims, batch, maxIters, tape, gout, gY, glam, stream); }
size_t proxtv_PD_TV_batched_tape_bytes(const int* ns, int nds, int npen, int batch, int maxIters) {
    return nd_tape_bytes_batched(ND_PD, ns, nds, npen, batch, maxIters); }
int proxtv_PD2_TV_batched_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_dev_f64", ND_PD2, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0,
                                (cudaStream_t)stream); }
int proxtv_PD2_TV_batched_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds, int npen,
                             int batch, int maxIters) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_f64", ND_PD2, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0, 0); }
int proxtv_PD2_TV_batched_record_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                        int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_record_dev_f64", ND_PD2, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                tape, tape_bytes, (cudaStream_t)stream); }
int proxtv_PD2_TV_batched_vjp_dev_f64(const int* ns, int nds, int npen, const double* dims, int batch, int maxIters, const void* tape,
                                     const double* gout, double* gY, double* glam, void* stream) {
    return dev_nd_vjp_batched<double>("proxtv_PD2_TV_batched_vjp_dev_f64", ND_PD2, ns, nds, npen, dims, batch, maxIters, tape, gout, gY, glam, stream); }
int proxtv_PD2_TV_batched_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_dev_f32", ND_PD2, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0,
                                (cudaStream_t)stream); }
int proxtv_PD2_TV_batched_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds, int npen,
                             int batch, int maxIters) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_f32", ND_PD2, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters, nullptr, 0, 0); }
int proxtv_PD2_TV_batched_record_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                        int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_record_dev_f32", ND_PD2, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                tape, tape_bytes, (cudaStream_t)stream); }
int proxtv_PD2_TV_batched_vjp_dev_f32(const int* ns, int nds, int npen, const double* dims, int batch, int maxIters, const void* tape,
                                     const float* gout, float* gY, double* glam, void* stream) {
    return dev_nd_vjp_batched<float>("proxtv_PD2_TV_batched_vjp_dev_f32", ND_PD2, ns, nds, npen, dims, batch, maxIters, tape, gout, gY, glam, stream); }
size_t proxtv_PD2_TV_batched_tape_bytes(const int* ns, int nds, int npen, int batch, int maxIters) {
    return nd_tape_bytes_batched(ND_PD2, ns, nds, npen, batch, maxIters); }

// ---- per-item penalties (DESIGN.md section 16.1) ----
int proxtv_PD_TV_batched_items_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns,
                                     int nds, int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_items_dev_f64", ND_PD, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, (cudaStream_t)stream, true); }
int proxtv_PD_TV_batched_items_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_items_f64", ND_PD, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, 0, true); }
int proxtv_PD_TV_batched_items_record_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns,
                                            int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<double>("proxtv_PD_TV_batched_items_record_dev_f64", ND_PD, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch,
                                maxIters, tape, tape_bytes, (cudaStream_t)stream, true); }
int proxtv_PD_TV_batched_items_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns,
                                     int nds, int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_items_dev_f32", ND_PD, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, (cudaStream_t)stream, true); }
int proxtv_PD_TV_batched_items_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_items_f32", ND_PD, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, 0, true); }
int proxtv_PD_TV_batched_items_record_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns,
                                            int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<float>("proxtv_PD_TV_batched_items_record_dev_f32", ND_PD, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch,
                                maxIters, tape, tape_bytes, (cudaStream_t)stream, true); }
int proxtv_PD2_TV_batched_items_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns,
                                     int nds, int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_items_dev_f64", ND_PD2, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, (cudaStream_t)stream, true); }
int proxtv_PD2_TV_batched_items_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_items_f64", ND_PD2, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, 0, true); }
int proxtv_PD2_TV_batched_items_record_dev_f64(const double* y, const double* lambdas, const double* dims, double* x, double* info, const int* ns,
                                            int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<double>("proxtv_PD2_TV_batched_items_record_dev_f64", ND_PD2, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch,
                                maxIters, tape, tape_bytes, (cudaStream_t)stream, true); }
int proxtv_PD2_TV_batched_items_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns,
                                     int nds, int npen, int batch, int maxIters, void* stream) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_items_dev_f32", ND_PD2, false, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, (cudaStream_t)stream, true); }
int proxtv_PD2_TV_batched_items_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns, int nds,
                                 int npen, int batch, int maxIters) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_items_f32", ND_PD2, true, false, y, lambdas, dims, x, info, ns, nds, npen, batch, maxIters,
                                nullptr, 0, 0, true); }
int proxtv_PD2_TV_batched_items_record_dev_f32(const float* y, const double* lambdas, const double* dims, float* x, double* info, const int* ns,
                                            int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, void* stream) {
    return run_pd_batched<float>("proxtv_PD2_TV_batched_items_record_dev_f32", ND_PD2, false, true, y, lambdas, dims, x, info, ns, nds, npen, batch,
                                maxIters, tape, tape_bytes, (cudaStream_t)stream, true); }
int proxtv_prox_fibers_lamf_dev_f64(const double* in, double* out, long long nf, int len, long long inc, const double* lamf, long long fpi, void* stream) {
    return dev_prox_fibers_lamf<double>("proxtv_prox_fibers_lamf_dev_f64", in, out, nf, len, inc, lamf, fpi, stream); }
int proxtv_fiber_tape_lamf_dev_f64(const double* y, long long nf, int len, long long inc, const double* lamf, long long fpi, unsigned* F, unsigned* U,
                                   void* stream) {
    return dev_tape_lamf<double>("proxtv_fiber_tape_lamf_dev_f64", y, nf, len, inc, lamf, fpi, F, U, stream); }
int proxtv_prox_fibers_lamf_dev_f32(const float* in, float* out, long long nf, int len, long long inc, const float* lamf, long long fpi, void* stream) {
    return dev_prox_fibers_lamf<float>("proxtv_prox_fibers_lamf_dev_f32", in, out, nf, len, inc, lamf, fpi, stream); }
int proxtv_fiber_tape_lamf_dev_f32(const float* y, long long nf, int len, long long inc, const float* lamf, long long fpi, unsigned* F, unsigned* U,
                                   void* stream) {
    return dev_tape_lamf<float>("proxtv_fiber_tape_lamf_dev_f32", y, nf, len, inc, lamf, fpi, F, U, stream); }

}  // extern "C"
