// emu_seq.cu -- TEST INFRASTRUCTURE: the sequential kernel (kernels_seq.cu, k_prox_seq) on the host.  taut_scan.cuh's Scan<T> is
// driven over every fiber of the slicing (nf, len, inc) -- fiber j starts at (j / inc) * inc * len + (j % inc), its weights at
// (j / inc) * inc * (len - 1) + (j % inc) -- in T arithmetic.  The float32 form is what the chunked, strided, sequential and
// long-fiber routes must reproduce bit for bit.  Not part of the product; built by tests/chunk_emu.py with nvcc (host code only).
#include "../../proxtv_b200/csrc/taut_scan.cuh"

using namespace ptv;

template <typename T>
static void seq_fibers(const T* A, T* X, long long nf, int n, long long inc, T lam, const T* lamv) {
    if (n <= 0) return;
    for (long long j = 0; j < nf; j++) {
        const long long base = (j / inc) * inc * n + (j % inc), wbase = (j / inc) * inc * (n - 1) + (j % inc);
        auto y = [&](int i) -> T { return A[base + (long long)i * inc]; };
        auto put = [&](int q, T v) { X[base + (long long)q * inc] = v; };
        auto run = [&](auto lamf) {
            Scan<T> s{};
            s.begin(0, y, lamf);
            int f, l; T v;
            while (s.i < n) {
                if (s.step(n, y, lamf, f, l, v) != K_NONE)
                    for (int q = f; q <= l; q++) put(q, v);
            }
            for (int q = s.last + 1; q < n; q++) put(q, s.lo);
        };
        if (lamv) {
            if (n == 1) { put(0, y(0)); continue; }
            auto ld = [&](int i) -> T { return lamv[wbase + (long long)i * inc]; };
            run(ArrayLam<T, decltype(ld)>{ld});
        } else {
            run(UniformLam<T>{lam});
        }
    }
}

extern "C" void emu_seq_fibers_f64(const double* A, double* X, long long nf, int n, long long inc, double lam, const double* lamv) {
    seq_fibers<double>(A, X, nf, n, inc, lam, lamv);
}
extern "C" void emu_seq_fibers_f32(const float* A, float* X, long long nf, int n, long long inc, float lam, const float* lamv) {
    seq_fibers<float>(A, X, nf, n, inc, lam, lamv);
}
