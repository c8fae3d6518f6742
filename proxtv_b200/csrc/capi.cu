// capi.cu -- the extern "C" boundary of libproxtv_b200.so (declared in include/proxtv_b200.h).
//
// Host-pointer entry points stage their arrays through a cached device arena (grow-only; one per process, guarded by a
// mutex), run the device-resident solver and copy the result back.  There is no CPU fallback: if no CUDA device is usable
// every entry point fails loudly.  Error behaviour follows the reference: "<fn>: <msg>" on stdout, info[RC] = RC_ERROR,
// return 0 (src/TV2Dopt.cpp:78-82,368-372).
#include "../../include/proxtv_b200.h"
#include "ptv_internal.h"
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
constexpr int MAX_DEV = 64;
Arena g_ws_d[MAX_DEV], g_io_d[MAX_DEV];
// slot of the current device; devices beyond MAX_DEV share the last slot's workspace tables only after have_device() refused them
int cur_dev() { int d = 0; if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); d = 0; } return (d < 0 || d >= MAX_DEV) ? MAX_DEV - 1 : d; }
#define g_ws (g_ws_d[cur_dev()])
#define g_io (g_io_d[cur_dev()])

// The workspaces, pipeline streams and captured graphs are one set per device, shared by every call: calls are serialised on the
// host by g_mu, and ON THE DEVICE by a per-device event -- a call's stream first waits for the previous call's work (which may
// have been enqueued on another stream), and records the event when its own work is enqueued.  Held for the whole call.
struct WsGuard {
    std::lock_guard<std::recursive_mutex> lk;
    cudaStream_t st; int dev;
    static cudaEvent_t& ev(int d) { static cudaEvent_t e[MAX_DEV] = {}; return e[d]; }
    explicit WsGuard(cudaStream_t s) : lk(g_mu), st(s), dev(-1) {
        int d = 0;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= MAX_DEV) { cudaGetLastError(); return; }
        dev = d;
        if (!ev(d)) { if (cudaEventCreateWithFlags(&ev(d), cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); ev(d) = nullptr; dev = -1; return; } }
        else cudaStreamWaitEvent(st, ev(d), 0);
    }
    ~WsGuard() { if (dev >= 0 && ev(dev)) cudaEventRecord(ev(dev), st); }
};

bool fail(const char* fn, const char* msg, double* info) {
    g_err = std::string(fn) + ": " + msg;
    printf("%s: %s\n", fn, msg); fflush(stdout);
    if (info) info[INFO_RC] = RC_ERROR;
    return false;
}
bool cuda_ok(const char* fn, cudaError_t e, double* info) {
    if (e == cudaSuccess) return true;
    cudaGetLastError();
    return fail(fn, (std::string("CUDA error: ") + cudaGetErrorString(e)).c_str(), info);
}
bool have_device(const char* fn, double* info) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) { cudaGetLastError();
        return fail(fn, "no usable CUDA device (libproxtv_b200 has no CPU fallback)", info); }
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= MAX_DEV - 1) { cudaGetLastError();
        return fail(fn, "current CUDA device index out of the supported range (0..62)", info); }
    return true;
}
inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

// Generic host-pointer batched 1D prox.  weights: nullptr or host array with nf*(len-1) entries.
template <typename T>
int host_prox_fibers(const char* fn, const T* in, T* out, long long nf, int len, long long inc, T lam, const T* lamv) {
    if (nf <= 0 || len <= 0) return 1;
    // the host arrays are staged as nf * len elements: with inc > 1 that is the whole slicing only when nf is a multiple of inc (the
    // last fibers of a partial slab would lie beyond it)
    if (inc < 1 || (inc > 1 && nf % inc != 0)) return fail(fn, "invalid fiber geometry (need inc >= 1 and nf a multiple of inc)", nullptr) ? 1 : 0;
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard(0);
    const size_t n = (size_t)nf * len, nw = lamv ? (size_t)nf * (len - 1) : 0;
    char* d = (char*)g_io.get(2 * al(n * sizeof(T)) + al(nw * sizeof(T) + 8));
    // scratch: staging of strided fibers (2n), or the overlapping tiles of contiguous fibers longer than shared memory
    T* scr = (inc != 1) ? (T*)g_ws.get(al((size_t)strided_scratch_elems(nf, len) * sizeof(T)))
                        : (len > 16384 && !lamv ? (T*)g_ws.get(al((size_t)lf_scratch_elems(nf, len) * sizeof(T)) + 256) : nullptr);
    if (!d) return fail(fn, "out of device memory", nullptr) ? 1 : 0;
    T* din = (T*)d; T* dout = (T*)(d + al(n * sizeof(T))); T* dw = (T*)(d + 2 * al(n * sizeof(T)));
    cudaStream_t st = 0;
    if (!cuda_ok(fn, cudaMemcpyAsync(din, in, n * sizeof(T), cudaMemcpyHostToDevice, st), nullptr)) return 0;
    if (nw && !cuda_ok(fn, cudaMemcpyAsync(dw, lamv, nw * sizeof(T), cudaMemcpyHostToDevice, st), nullptr)) return 0;
    FiberGeom g{nf, len, inc};
    long_fiber_note(-1);
    const Engine eng = (!lamv && nf >= 1024 && len >= 64) ? lane_guard<T>((Engine)g_engine, din, (long long)n, (double)lam, st) : (Engine)g_engine;
    if (!cuda_ok(fn, prox_fibers<T>(din, nullptr, IN_A, dout, 0, g, lam, lamv ? dw : nullptr, eng, scr, st,
                                     (inc == 1 && scr) ? lf_scratch_elems(nf, len) : (inc != 1 ? strided_scratch_elems(nf, len) : 0)), nullptr)) return 0;
    if (!cuda_ok(fn, cudaMemcpyAsync(out, dout, n * sizeof(T), cudaMemcpyDeviceToHost, st), nullptr)) return 0;
    if (!cuda_ok(fn, cudaStreamSynchronize(st), nullptr)) return 0;
    return 1;
}

template <typename T>
int host_dr2(const char* fn, size_t M, size_t N, int batch, const T* Y, T W1, T W2, T* out, int maxit, double* info) {
    if (!have_device(fn, info)) return 0;
    WsGuard guard(0);
    const size_t n = M * N * (size_t)batch;
    if (n == 0) { if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; } return 0; }
    char* d = (char*)g_io.get(2 * al(n * sizeof(T)));
    void* ws = g_ws.get(ws_bytes_dr2<T>(M, N, batch));
    if (!d || !ws) { fail(fn, "out of memory", info); return 0; }                       // TV2Dopt.cpp:383-384
    T* dY = (T*)d; T* dout = (T*)(d + al(n * sizeof(T)));
    cudaStream_t st = 0;
    if (!cuda_ok(fn, cudaMemcpyAsync(dY, Y, n * sizeof(T), cudaMemcpyHostToDevice, st), info)) return 0;
    double linfo[3] = {0, 0, RC_OK};                   // a NULL info must not hide a failed solve (nothing is copied back then)
    double* pinfo = info ? info : linfo;
    dr2_device<T>(M, N, batch, 0, dY, W1, W2, dout, maxit, pinfo, ws, (Engine)g_engine, st);
    if (pinfo[INFO_RC] == RC_ERROR) { fail(fn, "device solver failed", info); return 0; }
    if (!cuda_ok(fn, cudaMemcpyAsync(out, dout, n * sizeof(T), cudaMemcpyDeviceToHost, st), info)) return 0;
    if (!cuda_ok(fn, cudaStreamSynchronize(st), info)) return 0;
    return 0;
}

// DR2L1W_TV with host (host_io) or device arrays: `batch` images back to back, column-major (row_major = 0) or C order (1); W1:
// (M-1) x N, W2: M x (N-1) per image, laid out like Y (include/proxtv_b200.h).
template <typename T>
int run_drw(const char* fn, bool host_io, size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit,
            double* info, cudaStream_t st) {
    if (batch < 0) { fail(fn, "invalid shape (need batch >= 0)", info); return 0; }
    if (!have_device(fn, info)) return 0;
    WsGuard guard(st);
    const size_t n = M * N * (size_t)batch, n1 = M ? (M - 1) * N * (size_t)batch : 0, n2 = N ? M * (N - 1) * (size_t)batch : 0;
    if (n == 0) { if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; } return 0; }
    if (!Y || !out || (n1 && !W1) || (n2 && !W2)) { fail(fn, "NULL array", info); return 0; }
    void* ws = g_ws.get(ws_bytes_dr2<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", info); return 0; }                             // TV2DWopt.cpp:78-79
    if (!host_io) return drw_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, info, ws, (Engine)g_engine, st);
    char* d = (char*)g_io.get(2 * al(n * sizeof(T)) + al(n1 * sizeof(T) + 8) + al(n2 * sizeof(T) + 8));
    if (!d) { fail(fn, "out of memory", info); return 0; }
    T* dY = (T*)d; T* dout = (T*)(d + al(n * sizeof(T))); T* d1 = (T*)(d + 2 * al(n * sizeof(T))); T* d2 = (T*)((char*)d1 + al(n1 * sizeof(T) + 8));
    if (!cuda_ok(fn, cudaMemcpyAsync(dY, Y, n * sizeof(T), cudaMemcpyHostToDevice, st), info)) return 0;
    if (n1 && !cuda_ok(fn, cudaMemcpyAsync(d1, W1, n1 * sizeof(T), cudaMemcpyHostToDevice, st), info)) return 0;
    if (n2 && !cuda_ok(fn, cudaMemcpyAsync(d2, W2, n2 * sizeof(T), cudaMemcpyHostToDevice, st), info)) return 0;
    double linfo[3] = {0, 0, RC_OK};
    double* pinfo = info ? info : linfo;
    drw_device<T>(M, N, batch, row_major, dY, d1, d2, dout, maxit, pinfo, ws, (Engine)g_engine, st);
    if (pinfo[INFO_RC] == RC_ERROR) { fail(fn, "device solver failed", info); return 0; }
    if (!cuda_ok(fn, cudaMemcpyAsync(out, dout, n * sizeof(T), cudaMemcpyDeviceToHost, st), info)) return 0;
    if (!cuda_ok(fn, cudaStreamSynchronize(st), info)) return 0;
    return 0;
}

// CondatChambollePock2_TV with host (host_io) or device arrays: `batch` images back to back, column-major (row_major = 0) or C order
// (1); info: host, 3 doubles per image, or NULL.  Returns 1 on success, 0 on failure (src/TV2Dopt.cpp:600-602, :750-756).
template <typename T>
int run_cp2(const char* fn, bool host_io, size_t M, size_t N, int batch, int row_major, const T* Y, double lambda, T* X, int alg, int maxit,
            double* info, cudaStream_t st) {
    auto fail_all = [&](const char* msg) {          // msg nullptr: already reported
        if (msg) fail(fn, msg, info); else if (info) info[INFO_RC] = RC_ERROR;
        if (info) for (int b = 1; b < batch; b++) info[3 * (size_t)b + INFO_RC] = RC_ERROR;
        return 0;
    };
    if (alg != 0 && alg != 1 && alg != 2) return fail_all("Algorithm parameter has an invalid value");
    if (batch < 0) { fail(fn, "invalid shape (need batch >= 0)", info); return 0; }
    if (batch == 0) return 1;
    if (M < 1 || N < 1 || M > 0x7fffffff || N > 0x7fffffff) return fail_all("invalid shape (need 1 <= M, N < 2^31)");
    if (!Y || !X) return fail_all("NULL array");
    if (!have_device(fn, nullptr)) return fail_all(nullptr);
    WsGuard guard(st);
    const size_t n = M * N * (size_t)batch;
    void* ws = g_ws.get(ws_bytes_cp2(M, N, batch, sizeof(T)));
    if (!ws) return fail_all("out of memory");
    const T* dY = Y; T* dX = X;
    if (host_io) {
        char* d = (char*)g_io.get(2 * al(n * sizeof(T)));
        if (!d) return fail_all("out of memory");
        dY = (T*)d; dX = (T*)(d + al(n * sizeof(T)));
        if (!cuda_ok(fn, cudaMemcpyAsync((void*)dY, Y, n * sizeof(T), cudaMemcpyHostToDevice, st), nullptr)) return fail_all(nullptr);
    }
    std::vector<int> iters(info ? batch : 0);
    if (!cuda_ok(fn, cp2_device<T>(M, N, batch, row_major, dY, lambda, dX, alg, maxit, info ? iters.data() : nullptr, ws, st), nullptr))
        return fail_all(nullptr);
    if (host_io) {
        if (!cuda_ok(fn, cudaMemcpyAsync(X, dX, n * sizeof(T), cudaMemcpyDeviceToHost, st), nullptr)) return fail_all(nullptr);
        if (!cuda_ok(fn, cudaStreamSynchronize(st), nullptr)) return fail_all(nullptr);
    }
    if (info) for (int b = 0; b < batch; b++) { info[3 * (size_t)b + INFO_ITERS] = iters[b]; info[3 * (size_t)b + INFO_RC] = RC_OK; }
    return 1;
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
    if (!have_device(fn, info)) return 0;
    if (norms) for (int i = 0; i < npen; i++) if (norms[i] != 1.0) {
        fail(fn, "only p = 1 (TV-L1) penalty terms are implemented on the GPU path", info); return 0; }
    if (nds <= 0 || !ns) { fail(fn, "invalid dimensions", info); return 0; }
    NdTerms t;
    nd_terms(ns, nds, 0, nullptr, &t);                 // the element count; the solver checks the terms
    const long long n = t.n;
    WsGuard guard(st);
    scale_penalties(s, lambdas, npen);
    void* ws = g_ws.get(ws_bytes_pd<T>(n, npen));
    if (!ws) { fail(fn, "out of memory", info); return 0; }
    const T* dy = y; T* dx = x;
    if (host_io && n > 0) {
        char* d = (char*)g_io.get(2 * al((size_t)n * sizeof(T)));
        if (!d) { fail(fn, "out of memory", info); return 0; }
        dy = (T*)d; dx = (T*)(d + al((size_t)n * sizeof(T)));
        if (!cuda_ok(fn, cudaMemcpyAsync((void*)dy, y, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, st), info)) return 0;
    }
    if (!nd_solve<T>(s, dy, lambdas, dims, dx, info, ns, nds, npen, maxIters, ws, st, nullptr)) return 0;
    if (host_io && n > 0) {
        if (!cuda_ok(fn, cudaMemcpyAsync(x, dx, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, st), info)) return 0;
        if (!cuda_ok(fn, cudaStreamSynchronize(st), info)) return 0;
    }
    return 1;
}

template <typename T> static T* dev_scratch(long long nf, int len, long long inc) {
    if (nf <= 0 || len <= 0 || (inc == 1 && len <= 16384)) return nullptr;
    std::lock_guard<std::recursive_mutex> lk(g_mu);
    if (inc == 1) return (T*)g_ws.get(al((size_t)lf_scratch_elems(nf, len) * sizeof(T)) + 256);
    return (T*)g_ws.get(al((size_t)strided_scratch_elems(nf, len) * sizeof(T)));
}

// Backward pass of proxtv_prox_fibers_dev_*: refused calls write nothing; the scratch (chunked work only) comes from the workspace.
template <typename T>
static int dev_vjp(const char* fn, const T* y, const T* g, T* gx, T* gw, long long nf, int len, long long inc, T lam, const T* lamv,
                   void* stream) {
    if (nf < 0 || len < 0 || inc < 1) { fail(fn, "invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1)", nullptr); return 0; }
    if (nf == 0 || len == 0) return 1;
    if (!y || !g || !gx) { fail(fn, "NULL array", nullptr); return 0; }
    if (!lamv && !(lam >= 0)) { fail(fn, "negative penalty", nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    const size_t sb = ptvv::vjp_scratch_bytes(nf, len);
    void* scr = sb ? g_ws.get(sb) : nullptr;
    if (sb && !scr) { fail(fn, "out of device memory", nullptr); return 0; }
    return cuda_ok(fn, ptvv::vjp_fibers<T>(y, g, gx, gw, nf, len, inc, lam, lamv, scr, (cudaStream_t)stream), nullptr);
}

template <typename T>
static int dev_dr2(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, T W1, T W2, T* out, int maxit, double* info, void* stream) {
    if (!have_device(fn, info)) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = g_ws.get(ws_bytes_dr2<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", info); return 0; }
    return dr2_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, info, ws, (Engine)g_engine, (cudaStream_t)stream);
}

// Segmentation tape of y over the fibers (nf, len, inc) (nf a multiple of inc); refused calls write nothing.
template <typename T>
static int dev_tape(const char* fn, const T* y, long long nf, int len, long long inc, T lam, const T* lamv, uint32_t* F, uint32_t* U,
                    void* stream) {
    if (nf < 0 || len < 0 || inc < 1 || (nf > 0 && nf % inc != 0)) {
        fail(fn, "invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)", nullptr); return 0; }
    if (nf == 0 || len == 0) return 1;
    if (!y || !F || !U) { fail(fn, "NULL array", nullptr); return 0; }
    if (!lamv && !(lam >= 0)) { fail(fn, "negative penalty", nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    return cuda_ok(fn, ptvv::fiber_tape<T>(y, nf, len, inc, lam, lamv, F, U, (cudaStream_t)stream), nullptr);
}

template <typename T>
static int dev_vjp_tape(const char* fn, const uint32_t* F, const uint32_t* U, const T* g, T* gx, T* gw, long long nf, int len, long long inc,
                        void* stream) {
    if (nf < 0 || len < 0 || inc < 1 || (nf > 0 && nf % inc != 0)) {
        fail(fn, "invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)", nullptr); return 0; }
    if (nf == 0 || len == 0) return 1;
    if (!F || !U || !g || !gx) { fail(fn, "NULL array", nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    const size_t sb = ptvv::vjp_scratch_bytes(nf, len);
    void* scr = sb ? g_ws.get(sb) : nullptr;
    if (sb && !scr) { fail(fn, "out of device memory", nullptr); return 0; }
    return cuda_ok(fn, ptvv::vjp_fibers_tape<T>(F, U, g, gx, gw, nf, len, inc, scr, (cudaStream_t)stream), nullptr);
}

template <typename T>
static int dev_dr2_record(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, T W1, T W2, T* out, int maxit, void* tape,
                          size_t tape_bytes, double* info, void* stream) {
    if (M < 1 || N < 1 || batch < 1) { fail(fn, "invalid shape (need M, N, batch >= 1)", info); return 0; }
    if (!Y || !out || !tape) { fail(fn, "NULL array", info); return 0; }
    if (!(W1 >= 0) || !(W2 >= 0)) { fail(fn, "negative penalty", info); return 0; }
    if (tape_bytes < dr2_tape_bytes(M, N, batch, maxit)) { fail(fn, "tape_bytes smaller than proxtv_DR2_TV_tape_bytes()", info); return 0; }
    if (!have_device(fn, info)) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = g_ws.get(ws_bytes_dr2_record<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", info); return 0; }
    if (!cuda_ok(fn, dr2_record_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, tape, ws, (Engine)g_engine, (cudaStream_t)stream), info))
        return 0;
    if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; }
    return 1;
}

template <typename T>
static int dev_dr2_vjp(const char* fn, size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY,
                       double* glam, void* stream) {
    if (M < 1 || N < 1 || batch < 1) { fail(fn, "invalid shape (need M, N, batch >= 1)", nullptr); return 0; }
    if (!tape || !gout || !gY) { fail(fn, "NULL array", nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = dr2_tape_check(tape, sizeof(T), M, N, batch, row_major, maxit, (cudaStream_t)stream)) { fail(fn, why, nullptr); return 0; }
    void* ws = g_ws.get(ws_bytes_dr2_vjp<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", nullptr); return 0; }
    return cuda_ok(fn, dr2_vjp_device<T>(M, N, batch, row_major, maxit, tape, gout, gY, glam, ws, (cudaStream_t)stream), nullptr);
}

template <typename T>
static int dev_drw_record(const char* fn, size_t M, size_t N, int batch, int row_major, const T* Y, const T* W1, const T* W2, T* out, int maxit,
                          void* tape, size_t tape_bytes, double* info, void* stream) {
    if (M < 1 || N < 1 || batch < 1) { fail(fn, "invalid shape (need M, N, batch >= 1)", info); return 0; }
    if (!Y || !out || !tape || (M > 1 && !W1) || (N > 1 && !W2)) { fail(fn, "NULL array", info); return 0; }
    if (tape_bytes < drw_tape_bytes(M, N, batch, maxit)) { fail(fn, "tape_bytes smaller than proxtv_DR2L1W_TV_batched_tape_bytes()", info); return 0; }
    if (!have_device(fn, info)) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = g_ws.get(ws_bytes_drw_record<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", info); return 0; }
    if (!cuda_ok(fn, drw_record_device<T>(M, N, batch, row_major, Y, W1, W2, out, maxit, tape, ws, (Engine)g_engine, (cudaStream_t)stream), info))
        return 0;
    if (info) { info[INFO_ITERS] = maxit <= 0 ? MAX_ITERS_DR : maxit; info[INFO_RC] = RC_OK; }
    return 1;
}

template <typename T>
static int dev_drw_vjp(const char* fn, size_t M, size_t N, int batch, int row_major, int maxit, const void* tape, const T* gout, T* gY, T* gW1,
                       T* gW2, void* stream) {
    if (M < 1 || N < 1 || batch < 1) { fail(fn, "invalid shape (need M, N, batch >= 1)", nullptr); return 0; }
    if (!tape || !gout || !gY) { fail(fn, "NULL array", nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = drw_tape_check(tape, sizeof(T), M, N, batch, row_major, maxit, (cudaStream_t)stream)) { fail(fn, why, nullptr); return 0; }
    void* ws = g_ws.get(ws_bytes_drw_vjp<T>(M, N, batch));
    if (!ws) { fail(fn, "out of memory", nullptr); return 0; }
    return cuda_ok(fn, drw_vjp_device<T>(M, N, batch, row_major, maxit, tape, gout, gY, gW1, gW2, ws, (cudaStream_t)stream), nullptr);
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
    if (!y || !x || !lambdas || !dims || !ns || !tape) { fail(fn, "NULL array", info); return 0; }
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) { fail(fn, why, info); return 0; }
    for (int i = 0; i < npen; i++) if (!(lambdas[i] >= 0)) { fail(fn, "negative penalty", info); return 0; }
    const size_t need = nd_tape_bytes(s, ns, nds, npen, maxIters);
    if (need == 0) { fail(fn, "tape size does not fit in size_t (maxIters too large)", info); return 0; }
    if (tape_bytes < need) { fail(fn, too_small[s], info); return 0; }
    if (!have_device(fn, info)) return 0;
    WsGuard guard((cudaStream_t)stream);
    void* ws = g_ws.get(ws_bytes_pd<T>(t.n, npen));
    if (!ws) { fail(fn, "out of memory", info); return 0; }
    double linfo[3] = {0, 0, RC_OK};                   // the header needs the iteration count even when the caller passes no info
    double* pinfo = info ? info : linfo;
    scale_penalties(s, lambdas, npen);
    if (!nd_solve<T>(s, y, lambdas, dims, x, pinfo, ns, nds, npen, maxIters, ws, (cudaStream_t)stream, tape)) {
        fail(fn, "device solver failed", info); return 0; }
    return cuda_ok(fn, nd_tape_header(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, (int)pinfo[INFO_ITERS], (cudaStream_t)stream),
                   info) ? 1 : 0;
}

template <typename T>
static int dev_nd_vjp(const char* fn, NdSolver s, const int* ns, int nds, int npen, const double* dims, int maxIters, int iters,
                      const void* tape, const T* gout, T* gY, double* glam, void* stream) {
    if (!ns || !dims || !tape || !gout || !gY) { fail(fn, "NULL array", nullptr); return 0; }
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) { fail(fn, why, nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    if (const char* why = nd_tape_check(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, iters, (cudaStream_t)stream)) {
        fail(fn, why, nullptr); return 0; }
    void* ws = g_ws.get(ws_bytes_nd_vjp<T>(t, npen, glam != nullptr));
    if (!ws) { fail(fn, "out of memory", nullptr); return 0; }
    return cuda_ok(fn, nd_vjp_device<T>(s, t, npen, maxIters, iters, tape, gout, gY, glam, ws, (cudaStream_t)stream), nullptr);
}

// ---- batched PD_TV / PD2_TV (DESIGN.md section 16): `batch` items of prod(ns) elements back to back, each with its own stop rule ----
// Every refusal writes info[3 b + RC] = RC_ERROR for every item and nothing else; lambdas are never written (PD_TV's factor npen is
// applied to a copy).
static void mark_items(double* info, int batch) { if (info) for (int b = 0; b < batch; b++) info[3 * (size_t)b + INFO_RC] = RC_ERROR; }
static void fail_items(const char* fn, const char* msg, double* info, int batch) { fail(fn, msg, nullptr); mark_items(info, batch); }

// The solve (host_io: y and x are host arrays) or, given a tape, the recorded solve and then the tape's header and K table.
template <typename T>
static int run_pd_batched(const char* fn, NdSolver s, bool host_io, bool record, const T* y, const double* lambdas, const double* dims, T* x, double* info,
                          const int* ns, int nds, int npen, int batch, int maxIters, void* tape, size_t tape_bytes, cudaStream_t st) {
    static const char* const too_small[2] = {"tape_bytes smaller than proxtv_PD2_TV_batched_tape_bytes()",
                                             "tape_bytes smaller than proxtv_PD_TV_batched_tape_bytes()"};
    NdTerms t;
    if (record) {                                      // the order of the single-item record entry points
        if (!y || !x || !lambdas || !dims || !ns || !tape) { fail_items(fn, "NULL array", info, batch); return 0; }
        if (batch < 1) { fail_items(fn, "invalid batch (need batch >= 1)", info, batch); return 0; }
        if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) { fail_items(fn, why, info, batch); return 0; }
        for (int i = 0; i < npen; i++) if (!(lambdas[i] >= 0)) { fail_items(fn, "negative penalty", info, batch); return 0; }
        const size_t need = nd_tape_bytes(s, ns, nds, npen, maxIters, batch);
        if (need == 0) { fail_items(fn, "tape size does not fit in size_t (maxIters too large)", info, batch); return 0; }
        if (tape_bytes < need) { fail_items(fn, too_small[s], info, batch); return 0; }
        if (!have_device(fn, nullptr)) { mark_items(info, batch); return 0; }
    } else {                                           // the order of the single-item solve entry points
        if (!have_device(fn, nullptr)) { mark_items(info, batch); return 0; }
        if (nds <= 0 || !ns) { fail_items(fn, "invalid dimensions", info, batch); return 0; }
        if (batch < 1) { fail_items(fn, "invalid batch (need batch >= 1)", info, batch); return 0; }
        if (!y || !x || (npen > 0 && (!lambdas || !dims))) { fail_items(fn, "NULL array", info, batch); return 0; }
        if (s == ND_PD2 && npen > 2) { fail_items(fn, "this algorithm can not work with more than 2 penalties", info, batch); return 0; }
        if (s == ND_PD2 && npen < 1) { fail_items(fn, "invalid penalty dimensions", info, batch); return 0; }
        if (const char* why = nd_terms(ns, nds, npen, dims, &t)) { fail_items(fn, why, info, batch); return 0; }
    }
    const long long n = t.n;
    WsGuard guard(st);
    std::vector<double> lam(lambdas ? lambdas : nullptr, lambdas ? lambdas + (npen > 0 ? npen : 0) : nullptr);
    scale_penalties(s, lam.data(), npen);
    void* ws = g_ws.get(ws_bytes_pd<T>(n, npen, batch));
    if (!ws) { fail_items(fn, "out of memory", info, batch); return 0; }
    std::vector<double> linfo(3 * (size_t)batch);      // the tape's K table needs the rows even when the caller passes no info
    double* pinfo = info ? info : linfo.data();
    const size_t nt = (size_t)n * batch;
    const T* dy = y; T* dx = x;
    if (host_io && nt > 0) {
        char* d = (char*)g_io.get(2 * al(nt * sizeof(T)));
        if (!d) { fail_items(fn, "out of memory", info, batch); return 0; }
        dy = (T*)d; dx = (T*)(d + al(nt * sizeof(T)));
        if (!cuda_ok(fn, cudaMemcpyAsync((void*)dy, y, nt * sizeof(T), cudaMemcpyHostToDevice, st), nullptr)) { mark_items(info, batch); return 0; }
    }
    const int ok = s == ND_PD2 ? pd2_device<T>(dy, lam.data(), dims, dx, pinfo, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape, batch)
                               : pd_device<T>(dy, lam.data(), dims, dx, pinfo, ns, nds, npen, maxIters, ws, (Engine)g_engine, st, tape, batch);
    if (!ok) { fail_items(fn, "device solver failed", info, batch); return 0; }
    if (record && !cuda_ok(fn, nd_tape_header_batched(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, batch, pinfo, st), nullptr)) {
        mark_items(info, batch); return 0; }
    if (host_io && nt > 0) {
        if (!cuda_ok(fn, cudaMemcpyAsync(x, dx, nt * sizeof(T), cudaMemcpyDeviceToHost, st), nullptr) ||
            !cuda_ok(fn, cudaStreamSynchronize(st), nullptr)) { mark_items(info, batch); return 0; }
    }
    return 1;
}

template <typename T>
static int dev_nd_vjp_batched(const char* fn, NdSolver s, const int* ns, int nds, int npen, const double* dims, int batch, int maxIters,
                              const void* tape, const T* gout, T* gY, double* glam, void* stream) {
    if (!ns || !dims || !tape || !gout || !gY) { fail(fn, "NULL array", nullptr); return 0; }
    if (batch < 1) { fail(fn, "invalid batch (need batch >= 1)", nullptr); return 0; }
    NdTerms t;
    if (const char* why = nd_args_check(s, ns, nds, npen, dims, &t)) { fail(fn, why, nullptr); return 0; }
    if (!have_device(fn, nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    std::vector<int> K(batch);
    if (const char* why = nd_tape_check_batched(s, tape, sizeof(T), ns, nds, npen, dims, maxIters, batch, K.data(), (cudaStream_t)stream)) {
        fail(fn, why, nullptr); return 0; }
    void* ws = g_ws.get(ws_bytes_nd_vjp<T>(t, npen, glam != nullptr, batch));
    if (!ws) { fail(fn, "out of memory", nullptr); return 0; }
    return cuda_ok(fn, nd_vjp_device<T>(s, t, npen, maxIters, 0, tape, gout, gY, glam, ws, (cudaStream_t)stream, batch, K.data()), nullptr);
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
void proxtv_release_workspace(void) { std::lock_guard<std::recursive_mutex> lk(g_mu); for (int d = 0; d < MAX_DEV; d++) { g_ws_d[d].release(); g_io_d[d].release(); } }

// ---- experimental: the lane-per-fiber streaming engine (kernels_lane.cu), device pointers ----
int proxtv_lane_prox_dev_f64(int op, const double* A, const double* B, const double* C, double* X, long long nf, int len, long long inc,
                             double lam, void* stream) {
    WsGuard guard((cudaStream_t)stream);
    void* scr = ptvl::lane_scratch(nf, len);
    if (!scr) return 0;
    cudaError_t e = ptvl::lane_prox<double>(op, A, B, C, X, nf, len, inc, lam, scr, (cudaStream_t)stream);
    if (e != cudaSuccess) { cudaGetLastError(); g_err = std::string("proxtv_lane_prox_dev_f64: ") + cudaGetErrorString(e); return 0; }
    return 1;
}
int proxtv_lane_prox2_dev_f64(int op, const double* A, const double* B, const double* C, double* X, double* X2, long long nf, int len, long long inc,
                              double lam, void* stream) {
    WsGuard guard((cudaStream_t)stream);
    void* scr = ptvl::lane_scratch(nf, len);
    if (!scr) return 0;
    cudaError_t e = ptvl::lane_prox<double>(op, A, B, C, X, nf, len, inc, lam, scr, (cudaStream_t)stream, X2);
    if (e != cudaSuccess) { cudaGetLastError(); g_err = std::string("proxtv_lane_prox2_dev_f64: ") + cudaGetErrorString(e); return 0; }
    return 1;
}
int proxtv_lane_prox_dev_f32(int op, const float* A, const float* B, const float* C, float* X, long long nf, int len, long long inc,
                             float lam, void* stream) {
    WsGuard guard((cudaStream_t)stream);
    void* scr = ptvl::lane_scratch(nf, len);
    if (!scr) return 0;
    cudaError_t e = ptvl::lane_prox<float>(op, A, B, C, X, nf, len, inc, lam, scr, (cudaStream_t)stream);
    if (e != cudaSuccess) { cudaGetLastError(); g_err = std::string("proxtv_lane_prox_dev_f32: ") + cudaGetErrorString(e); return 0; }
    return 1;
}
void proxtv_lane_tuning(int clen, int halo, int variant) { ptvl::lane_set_tuning(clen, halo, variant); }
void proxtv_lane_tasklog(unsigned long long* dev, long long cap_tasks) { ptvl::lane_set_tasklog(dev, cap_tasks); }
int proxtv_lane_guard_last(void) { return lane_guard_last(); }
int proxtv_long_fiber_last(void) { return long_fiber_last(); }
unsigned long long proxtv_lane_stats(int reset) { return ptvl::lane_read_stats(reset); }

// ---- Part 1: drop-in symbols ----
void hybridTautString_TV1(double* y, int n, double lambda, double* x) {
    host_prox_fibers<double>("hybridTautString_TV1", y, x, 1, n, 1, lambda, nullptr);
}
void hybridTautString_TV1_custom(double* y, int n, double lambda, double* x, double) {
    host_prox_fibers<double>("hybridTautString_TV1_custom", y, x, 1, n, 1, lambda, nullptr);
}
int classicTautString_TV1(double* signal, int n, double lam, double* prox) {
    if (n <= 0) return 1;
    if (lam <= 0 || n == 1) { memmove(prox, signal, (size_t)n * sizeof(double)); return 1; }   // TVL1opt_tautstring.cpp:258-263
    host_prox_fibers<double>("classicTautString_TV1", signal, prox, 1, n, 1, lam, nullptr);
    return 1;
}
int linearizedTautString_TV1(double* y, double lambda, double* x, int n) {
    host_prox_fibers<double>("linearizedTautString_TV1", y, x, 1, n, 1, lambda, nullptr);
    return 1;
}
void TV1D_denoise(double* input, double* output, const int width, const double lambda) {
    if (width > 0 && lambda >= 0) host_prox_fibers<double>("TV1D_denoise", input, output, 1, width, 1, lambda, nullptr);
}
int tautString_TV1_Weighted(double* y, double* lambda, double* x, int n) {
    if (n == 1) { x[0] = y[0]; return 1; }
    host_prox_fibers<double>("tautString_TV1_Weighted", y, x, 1, n, 1, 0.0, lambda);
    return 1;
}
// The reference's alternative 1D TV-L1 solvers compute the same unique minimiser (<= 4e-14 apart on random data, 9e-7 for Condat's
// float-truncating taut-string variant -- measured with the compiled reference): they all map onto the exact kernel.
static void ok_info(double* info) { if (info) { info[INFO_ITERS] = 0; info[INFO_GAP] = 0; info[INFO_RC] = RC_OK; } }
int PN_TV1(double* y, double lambda, double* x, double* info, int n, double, void*) {
    if (!host_prox_fibers<double>("PN_TV1", y, x, 1, n, 1, lambda, nullptr)) { if (info) info[INFO_RC] = RC_ERROR; return 0; }
    ok_info(info); return 1;
}
int PN_TV1_Weighted(double* Y, double* W, double* X, double* info, int n, double, void*) {
    if (n == 1) { X[0] = Y[0]; ok_info(info); return 1; }
    if (!host_prox_fibers<double>("PN_TV1_Weighted", Y, X, 1, n, 1, 0.0, W)) { if (info) info[INFO_RC] = RC_ERROR; return 0; }
    ok_info(info); return 1;
}
void TV1D_denoise_tautstring(double* input, double* output, int width, const double lambda) {
    if (width > 0 && lambda >= 0) host_prox_fibers<double>("TV1D_denoise_tautstring", input, output, 1, width, 1, lambda, nullptr);
}
void SolveTVConvexQuadratic_a1_nw(int n, double* b, double w, double* solution) {
    host_prox_fibers<double>("SolveTVConvexQuadratic_a1_nw", b, solution, 1, n, 1, w, nullptr);
}
void SolveTVConvexQuadratic_a1(int n, double* b, double* w, double* solution) {
    if (n == 1) { solution[0] = b[0]; return; }
    host_prox_fibers<double>("SolveTVConvexQuadratic_a1", b, solution, 1, n, 1, 0.0, w);
}
void dp(int n, double* y, double lam, double* beta) {
    host_prox_fibers<double>("dp", y, beta, 1, n, 1, lam, nullptr);
}
int TV(double* y, double lambda, double* x, double* info, int n, double p, void*) {
    if (p < 1) { fail("TVopt", "TV only works for norms p >= 1", info); return 0; }                // TVgenopt.cpp:37-38
    if (p != 1) { fail("TVopt", "only p = 1 (TV-L1) is implemented on the GPU path", info); return 0; }
    if (!host_prox_fibers<double>("TVopt", y, x, 1, n, 1, lambda, nullptr)) { if (info) info[INFO_RC] = RC_ERROR; return 0; }
    if (info) { info[INFO_RC] = RC_OK; info[INFO_ITERS] = 0; info[INFO_GAP] = 0; }                 // :43-47
    return 1;
}
int DR2_TV(size_t M, size_t N, double* unary, double W1, double W2, double norm1, double norm2, double* s, int, int maxit,
           double* info) {
    if (norm1 != 1.0 || norm2 != 1.0) { fail("DR2_TV", "only p = 1 (TV-L1) penalties are implemented on the GPU path", info); return 0; }
    return host_dr2<double>("DR2_TV", M, N, 1, unary, W1, W2, s, maxit, info);
}
int DR2L1W_TV(size_t M, size_t N, double* unary, double* W1, double* W2, double* s, int, int maxit, double* info) {
    return run_drw<double>("DR2L1W_TV", true, M, N, 1, 0, unary, W1, W2, s, maxit, info, 0);
}
int CondatChambollePock2_TV(size_t M, size_t N, double* Y, double lambda, double* X, short alg, int maxit, double* info) {
    return run_cp2<double>("Condat2_TV", true, M, N, 1, 0, Y, lambda, X, alg, maxit, info, 0);
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
    if (!have_device("proxtv_prox_fibers_dev_f64", nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    long_fiber_note(-1);
    const Engine eng = (!lamv && nf >= 1024 && len >= 64) ? lane_guard<double>((Engine)g_engine, in, nf * (long long)len, lam, (cudaStream_t)stream) : (Engine)g_engine;
    return cuda_ok("proxtv_prox_fibers_dev_f64", prox_fibers<double>(in, nullptr, IN_A, out, 0, FiberGeom{nf, len, inc}, lam, lamv, eng, dev_scratch<double>(nf, len, inc), (cudaStream_t)stream,
                                                                 (inc == 1 && len > 16384) ? lf_scratch_elems(nf, len) : (inc != 1 ? strided_scratch_elems(nf, len) : 0)), nullptr);
}
int proxtv_prox_fibers_dev_f32(const float* in, float* out, long long nf, int len, long long inc, float lam, const float* lamv, void* stream) {
    if (!have_device("proxtv_prox_fibers_dev_f32", nullptr)) return 0;
    WsGuard guard((cudaStream_t)stream);
    long_fiber_note(-1);
    const Engine eng = (!lamv && nf >= 1024 && len >= 64) ? lane_guard<float>((Engine)g_engine, in, nf * (long long)len, (double)lam, (cudaStream_t)stream) : (Engine)g_engine;
    return cuda_ok("proxtv_prox_fibers_dev_f32", prox_fibers<float>(in, nullptr, IN_A, out, 0, FiberGeom{nf, len, inc}, lam, lamv, eng, dev_scratch<float>(nf, len, inc), (cudaStream_t)stream,
                                                                 (inc == 1 && len > 16384) ? lf_scratch_elems(nf, len) : (inc != 1 ? strided_scratch_elems(nf, len) : 0)), nullptr);
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
    return host_prox_fibers<double>("proxtv_prox_fibers_f64", in, out, nf, len, inc, lam, lamv);
}
int proxtv_prox_fibers_f32(const float* in, float* out, long long nf, int len, long long inc, float lam, const float* lamv) {
    return host_prox_fibers<float>("proxtv_prox_fibers_f32", in, out, nf, len, inc, lam, lamv);
}

int proxtv_DR2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double W1, double W2, double* out, int maxit, double* info, void* stream) {
    return dev_dr2<double>("proxtv_DR2_TV_dev_f64", M, N, batch, row_major, Y, W1, W2, out, maxit, info, stream); }
int proxtv_DR2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, float W1, float W2, float* out, int maxit, double* info, void* stream) {
    return dev_dr2<float>("proxtv_DR2_TV_dev_f32", M, N, batch, row_major, Y, W1, W2, out, maxit, info, stream); }
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
    return host_dr2<double>("proxtv_DR2_TV_batched_f64", M, N, batch, Y, W1, W2, out, maxit, info); }
int proxtv_DR2_TV_batched_f32(size_t M, size_t N, int batch, const float* Y, float W1, float W2, float* out, int maxit, double* info) {
    return host_dr2<float>("proxtv_DR2_TV_batched_f32", M, N, batch, Y, W1, W2, out, maxit, info); }

int proxtv_CP2_TV_dev_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double lambda, double* X, int alg, int maxit,
                          double* info, void* stream) {
    return run_cp2<double>("proxtv_CP2_TV_dev_f64", false, M, N, batch, row_major, Y, lambda, X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2_TV_dev_f32(size_t M, size_t N, int batch, int row_major, const float* Y, double lambda, float* X, int alg, int maxit,
                          double* info, void* stream) {
    return run_cp2<float>("proxtv_CP2_TV_dev_f32", false, M, N, batch, row_major, Y, lambda, X, alg, maxit, info, (cudaStream_t)stream); }
int proxtv_CP2_TV_batched_f64(size_t M, size_t N, int batch, int row_major, const double* Y, double lambda, double* X, int alg, int maxit,
                              double* info) {
    return run_cp2<double>("proxtv_CP2_TV_batched_f64", true, M, N, batch, row_major, Y, lambda, X, alg, maxit, info, 0); }
int proxtv_CP2_TV_batched_f32(size_t M, size_t N, int batch, int row_major, const float* Y, double lambda, float* X, int alg, int maxit,
                              double* info) {
    return run_cp2<float>("proxtv_CP2_TV_batched_f32", true, M, N, batch, row_major, Y, lambda, X, alg, maxit, info, 0); }

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

}  // extern "C"
