// emu_vjp_tape.cu -- TEST INFRASTRUCTURE: the tape-driven form of the backward kernels' three passes (vjp.cu with TAPE, logic in
// proxtv_b200/csrc/vjp_core.cuh: VjpScan::step, vjp_carry_from, vjp_fix_chunk_sg) run on the CPU with a given chunk length, item by item
// in the order the device leaves them, and the tape encoder (vjp_tape_edge).  Not part of the product; built by tests/dr2_vjp_emu.py
// with g++ (host code only; the CUDA headers only supply the __host__ __device__ macros).
#include "../../proxtv_b200/csrc/vjp_core.cuh"
#include <vector>

using namespace ptvv;

template <typename T> struct HostOut {
    T* px; T* pw; long long xb, wb, inc;
    void gx(int k, T v) { px[xb + (long long)k * inc] = v; }
    void gw(int e, T v) { if (pw) pw[wb + (long long)e * inc] = v; }
};

template <typename T>
static void tape(const T* y, long long nf, int len, long long inc, double lam, const T* w, uint32_t* F, uint32_t* U) {
    const long long n = nf * (long long)len, nw = (long long)(vjp_tape_set_bytes(n) / 4);
    for (long long q = 0; q < nw; q++) { F[q] = 0; U[q] = 0; }
    for (long long i = 0; i < n; i++) {
        uint32_t f = 0, u = 0;
        vjp_tape_edge<T>(y, i, len, inc, lam, w, f, u);
        F[i >> 5] |= f << (i & 31); U[i >> 5] |= u << (i & 31);
    }
}

template <typename T>
static void run(const uint32_t* F, const uint32_t* U, const T* g, T* gx, T* gw, long long nf, int len, long long inc, int C) {
    if (nf <= 0 || len <= 0) return;
    if (C <= 0 || C > len) C = len;
    const int nc = (len + C - 1) / C;
    std::vector<VjpRec> rec((size_t)(nf * nc));
    std::vector<VjpMeans> mm((size_t)(nf * nc));
    auto base = [&](long long f) { return (f / inc) * inc * (long long)len + f % inc; };
    auto wbase = [&](long long f) { return (f / inc) * inc * (long long)(len - 1) + f % inc; };
    for (int c = 0; c < nc; c++)
        for (long long f = 0; f < nf; f++) {
            const long long xb = base(f), wb = wbase(f);
            const int c0 = c * C, c1 = c0 + C < len ? c0 + C : len;
            HostOut<T> out{gx, gw, xb, wb, inc};
            VjpScan<T> sc;
            sc.begin(c0, len, T(0), c0 > 0 && vjp_tape_fused(F, U, xb + (long long)(c0 - 1) * inc));
            for (int i = c0; i < c1; i++) {
                const long long e = xb + (long long)i * inc;
                const bool nl = i + 1 < len;
                sc.step(i, g[e], nl && vjp_tape_fused(F, U, e), [&]() { return vjp_tape_sgn(F, U, e); }, out);
            }
            sc.finish(rec[f * nc + c]);
        }
    if (nc == 1) return;
    for (int c = nc - 1; c >= 0; c--)
        for (long long f = 0; f < nf; f++) {
            const long long xb = base(f);
            vjp_carry_from<T>(&rec[f * nc], c, nc, C, len, [&](int i) { return g[xb + (long long)i * inc]; },
                              [&](int k) -> VjpMeans& { return mm[f * nc + k]; });
        }
    for (int c = 0; c < nc; c++)
        for (long long f = 0; f < nf; f++) {
            const long long xb = base(f), ri = f * nc + c;
            const int c0 = c * C, c1 = c0 + C < len ? c0 + C : len;
            HostOut<T> out{gx, gw, xb, wbase(f), inc};
            const double mnext = c + 1 < nc ? vjp_first_mean(rec[ri + 1], mm[ri + 1]) : 0.0;
            vjp_fix_chunk_sg<T>(rec[ri], mm[ri], c0, c1, len, mnext, gw != nullptr,
                                [&](int e) { return vjp_tape_sgn(F, U, xb + (long long)e * inc); },
                                [&](int i) { return gx[xb + (long long)i * inc]; }, out);
        }
}

extern "C" {
void emu_tape_f64(const double* y, long long nf, int len, long long inc, double lam, const double* w, uint32_t* F, uint32_t* U) {
    tape<double>(y, nf, len, inc, lam, w, F, U);
}
void emu_tape_f32(const float* y, long long nf, int len, long long inc, float lam, const float* w, uint32_t* F, uint32_t* U) {
    tape<float>(y, nf, len, inc, (double)lam, w, F, U);
}
void emu_vjp_tape_f64(const uint32_t* F, const uint32_t* U, const double* g, double* gx, double* gw, long long nf, int len, long long inc,
                      int chunk) {
    run<double>(F, U, g, gx, gw, nf, len, inc, chunk);
}
void emu_vjp_tape_f32(const uint32_t* F, const uint32_t* U, const float* g, float* gx, float* gw, long long nf, int len, long long inc,
                      int chunk) {
    run<float>(F, U, g, gx, gw, nf, len, inc, chunk);
}
}
