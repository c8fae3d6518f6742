// emu_vjp.cu -- TEST INFRASTRUCTURE: runs proxtv_b200/csrc/vjp_core.cuh (the three passes of the backward kernels in vjp.cu: chunk
// scan, carry, fix-up) on the CPU with a given chunk length, item by item in the order the device leaves them (every pass 1 before pass
// 2, every pass 2 before pass 3).  Not part of the product; built by tests/vjp_emu.py with g++ (host code only; the CUDA headers only
// supply the __host__ __device__ macros).
#include "../../proxtv_b200/csrc/vjp_core.cuh"
#include <vector>

using namespace ptvv;

template <typename T> struct HostOut {
    T* px; T* pw; long long xb, wb, inc;
    void gx(int k, T v) { px[xb + (long long)k * inc] = v; }
    void gw(int e, T v) { if (pw) pw[wb + (long long)e * inc] = v; }
};

template <typename T>
static void run(const T* y, const T* g, T* gx, T* gw, long long nf, int len, long long inc, double lam, const T* w, int C) {
    if (nf <= 0 || len <= 0) return;
    if (C <= 0 || C > len) C = len;
    const int nc = (len + C - 1) / C;
    std::vector<VjpRec> rec((size_t)(nf * nc));
    std::vector<VjpMeans> mm((size_t)(nf * nc));
    auto base = [&](long long f) { return (f / inc) * inc * (long long)len + f % inc; };
    auto wbase = [&](long long f) { return (f / inc) * inc * (long long)(len - 1) + f % inc; };
    auto wpos = [&](long long wb, int e) { return w ? w[wb + (long long)e * inc] > T(0) : lam > 0.0; };
    for (int c = 0; c < nc; c++)
        for (long long f = 0; f < nf; f++) {
            const long long xb = base(f), wb = wbase(f);
            const int c0 = c * C, c1 = c0 + C < len ? c0 + C : len;
            HostOut<T> out{gx, gw, xb, wb, inc};
            VjpScan<T> sc;
            const T y0 = y[xb + (long long)c0 * inc];
            sc.begin(c0, len, y0, c0 > 0 && y[xb + (long long)(c0 - 1) * inc] == y0 && wpos(wb, c0 - 1));
            for (int i = c0; i < c1; i++) {
                const bool nl = i + 1 < len;
                sc.row(i, g[xb + (long long)i * inc], nl ? y[xb + (long long)(i + 1) * inc] : T(0), nl && wpos(wb, i), out);
            }
            sc.finish(rec[f * nc + c]);
        }
    if (nc == 1) return;
    for (int c = nc - 1; c >= 0; c--)                    // any order: the open segments are disjoint (backwards here, to show it)
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
            vjp_fix_chunk<T>(rec[ri], mm[ri], c0, c1, len, mnext, gw != nullptr, [&](int i) { return y[xb + (long long)i * inc]; },
                             [&](int i) { return gx[xb + (long long)i * inc]; }, out);
        }
}

extern "C" {
void emu_vjp_f64(const double* y, const double* g, double* gx, double* gw, long long nf, int len, long long inc, double lam, const double* w,
                 int chunk) {
    run<double>(y, g, gx, gw, nf, len, inc, lam, w, chunk);
}
void emu_vjp_f32(const float* y, const float* g, float* gx, float* gw, long long nf, int len, long long inc, float lam, const float* w,
                 int chunk) {
    run<float>(y, g, gx, gw, nf, len, inc, (double)lam, w, chunk);
}
}
