// cp2.cu -- CondatChambollePock2_TV (src/TV2Dopt.cpp:587-760): the 2D TV-L1 prox by Condat's (alg 0), Chambolle-Pock's (alg 1) and
// the accelerated Chambolle-Pock (alg 2) primal-dual iteration, for `batch` independent images, device-resident (DESIGN.md section 15).
//
// Each iteration is one fused stencil launch over all images.  A block owns a 32 x 32 tile of one image: it recomputes the primal step
// Xt and the extrapolation Z = Xt + theta (Xt - X) on the tile plus a one-cell halo on its high side (the dual steps need Z one cell
// further along each axis), keeps Z in shared memory, writes the tile's X' and clipped duals U' into the other buffer of a ping-pong
// pair (neighbouring tiles still read the old ones), and adds the tile's float64 sums of (Xt - X)^2 and X^2 to its image's stop sums.
// The next launch decides each image's stop test (sqrt(num / den) > 0, STOP_CONDAT = 0) from the sums that stream order has already
// completed; an image that stops does nothing in later launches, and the launch that finds it stopped records its iteration count.
// The step sizes depend only on the iteration number (and lambda for alg 2), so the host computes them in float64 in the reference's
// order and passes them to each launch; float32 solves round each value once.
//
// Storage: both memory orders of an M x N image are an F x S array with the F axis contiguous (column-major: F = M, S = N;
// row-major: F = N, S = M); only the roles of the two difference terms swap, and D = a + b is commutative in IEEE arithmetic, so
// both orders give the same bits.  The duals are stored padded to F x S (the last row of Uf, the last column of Us unused).
//
// Weighted (DESIGN.md section 15.1, alg 0 and 1 only): each dual is clipped to its own edge's weight instead of lambda.  The caller's
// maps are read in place: in F x S terms they are an (F-1) x S map Wf of the edges along F and an F x (S-1) map Ws of the edges
// along S, both F-contiguous (column-major: Wf = W1, Ws = W2; C order: Wf = W2, Ws = W1), so the weight of the dual at q = b F S +
// f + F s is Wf[q - (b S + s)] and Ws[q - b F].
//
// Recorded (DESIGN.md section 15.2): given a tape, one more launch after k_cp2_out writes the fused-edge tape of the backward
// (cp2_vjp.cu) from the final duals; every launch before it is the same.
#include "ptv_internal.h"
#include <math.h>
#include <stdio.h>

namespace ptv {

namespace {

constexpr int TF = 32, TS = 32;                     // tile (contiguous axis x strided axis)
constexpr int HF = TF + 1, HS = TS + 1;             // with the high-side halo
constexpr int THREADS = 256;
constexpr int CELLS = HF * HS;
constexpr int PER = (CELLS + THREADS - 1) / THREADS;
constexpr int SLOTS = 8;                            // partial-sum addresses per image (spreads the atomics of one image's tiles)
constexpr int ITERS_PER_CHECK = 64;                 // launches between two reads of the running-image count

static inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct Geom {
    int F, S;             // contiguous and strided extent of one image
    long long img;        // elements per image
    int ntf, tiles;       // tiles along F, tiles per image
    int batch;
};

template <typename T> __device__ __forceinline__ T clip(T v, T lam) { return v < -lam ? -lam : (v > lam ? lam : v); }

// sums: [3][batch][SLOTS][2] (num, den), slot set it % 3 is written by iteration it.  stopped[b]: 0 while image b runs, else the
// reference's final `it` (iterations run + 1).
__device__ __forceinline__ bool keeps_running(const double* sums, int batch, int b, int slot) {
    const double* sp = sums + ((size_t)slot * batch + b) * SLOTS * 2;
    double num = 0, den = 0;
    for (int k = 0; k < SLOTS; k++) { num += sp[2 * k]; den += sp[2 * k + 1]; }
    return sqrt(num / den) > 0;
}

// WTD: clip each dual to its edge's weight in Wf / Ws (lam unused); else to lam (Wf, Ws unused)
template <typename T, bool WTD>
__global__ void __launch_bounds__(THREADS, 3) k_cp2_iter(Geom g, const T* __restrict__ Y, const T* __restrict__ X,
                                                         const T* __restrict__ Uf, const T* __restrict__ Us, T* __restrict__ Xn,
                                                         T* __restrict__ Ufn, T* __restrict__ Usn, int* stopped, double* sums, int it, int alg, T tau, T c, T theta, T sigma, T lam,
                                                         const T* __restrict__ Wf, const T* __restrict__ Ws) {
    __shared__ T zs[CELLS];
    __shared__ double red[THREADS / 32][2];
    const int tid = threadIdx.x;
    const int tile = blockIdx.x, f0 = (tile % g.ntf) * TF, s0 = (tile / g.ntf) * TS;
    const int F = g.F, S = g.S;
    for (int b = blockIdx.y; b < g.batch; b += gridDim.y) {
        if (stopped[b]) continue;
        if (it > 1 && !keeps_running(sums, g.batch, b, (it - 1) % 3)) {          // the loop test of iteration it
            if (tile == 0 && tid == 0) stopped[b] = it;
            continue;
        }
        if (tile == 0 && tid < 2 * SLOTS) sums[((size_t)((it + 1) % 3) * g.batch + b) * SLOTS * 2 + tid] = 0;
        const long long base = (long long)b * g.img;
        T zv[PER], ufv[PER], usv[PER];
        double num = 0, den = 0;
#pragma unroll
        for (int k = 0; k < PER; k++) {
            const int p = tid + k * THREADS;
            const int lf = p % HF, ls = p / HF, f = f0 + lf, s = s0 + ls;
            zv[k] = ufv[k] = usv[k] = 0;
            if (p >= CELLS || f >= F || s >= S) continue;
            const long long q = base + f + (long long)F * s;
            const T x = X[q], y = Y[q];
            const T uf = f < F - 1 ? Uf[q] : T(0), us = s < S - 1 ? Us[q] : T(0);
            T D;
            const T tf = F == 1 ? T(0) : (f == 0 ? -uf : (f == F - 1 ? Uf[q - 1] : Uf[q - 1] - uf));
            const T ts = S == 1 ? T(0) : (s == 0 ? -us : (s == S - 1 ? Us[q - F] : Us[q - F] - us));
            D = (F > 1 && S > 1) ? tf + ts : (F > 1 ? tf : ts);
            const T xt = alg == 0 ? x - tau * ((x - y) + D) : c * (x + tau * (y - D));
            const T z = xt + theta * (xt - x);
            zs[p] = z;
            if (lf < TF && ls < TS) {
                Xn[q] = xt;
                const double d = (double)xt - (double)x;
                num += d * d; den += (double)x * (double)x;
                zv[k] = z; ufv[k] = uf; usv[k] = us;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PER; k++) {
            const int p = tid + k * THREADS;
            const int lf = p % HF, ls = p / HF, f = f0 + lf, s = s0 + ls;
            if (p >= CELLS || lf >= TF || ls >= TS || f >= F || s >= S) continue;
            const long long q = base + f + (long long)F * s;
            if (f < F - 1) Ufn[q] = clip<T>(ufv[k] + sigma * (zs[p + 1] - zv[k]), WTD ? Wf[q - ((long long)b * S + s)] : lam);
            if (s < S - 1) Usn[q] = clip<T>(usv[k] + sigma * (zs[p + HF] - zv[k]), WTD ? Ws[q - (long long)b * F] : lam);
        }
        for (int o = 16; o > 0; o >>= 1) { num += __shfl_down_sync(0xffffffffu, num, o); den += __shfl_down_sync(0xffffffffu, den, o); }
        if ((tid & 31) == 0) { red[tid >> 5][0] = num; red[tid >> 5][1] = den; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < THREADS / 32; w++) { num += red[w][0]; den += red[w][1]; }
            double* sp = sums + (((size_t)(it % 3) * g.batch + b) * SLOTS + tile % SLOTS) * 2;
            atomicAdd(sp, num); atomicAdd(sp + 1, den);
        }
        __syncthreads();                                                       // zs and red are reused by the next image
    }
}

// X = Y, Uf = Y(f+1, s) - Y(f, s), Us = Y(f, s+1) - Y(f, s)
template <typename T>
__global__ void k_cp2_init(Geom g, const T* __restrict__ Y, T* __restrict__ X, T* __restrict__ Uf, T* __restrict__ Us) {
    const long long n = g.img * g.batch;
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const long long e = q % g.img;
        const int f = (int)(e % g.F), s = (int)(e / g.F);
        const T y = Y[q];
        X[q] = y;
        if (f < g.F - 1) Uf[q] = Y[q + 1] - y;
        if (s < g.S - 1) Us[q] = Y[q + g.F] - y;
    }
}

// how many images still run after iteration it
__global__ void k_cp2_alive(const int* stopped, const double* sums, int batch, int it, int* alive) {
    int n = 0;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) n += !stopped[b] && keeps_running(sums, batch, b, it % 3);
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    __shared__ int r[32];
    if ((threadIdx.x & 31) == 0) r[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) { for (int w = 1; w < (int)(blockDim.x >> 5); w++) n += r[w]; *alive = n; }
}

// the result of each image from the buffer its last iteration wrote; images still running when the loop ended stop at it_end
template <typename T>
__global__ void k_cp2_out(Geom g, const T* __restrict__ X0, const T* __restrict__ X1, int* stopped, int it_end, T* __restrict__ out) {
    const long long n = g.img * g.batch;
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(q / g.img);
        const int st = stopped[b] ? stopped[b] : it_end;
        out[q] = ((st - 1) & 1) ? X1[q] : X0[q];
    }
}

int grid_1d(long long n) { long long b = (n + 255) / 256; return (int)(b < 132 * 16 ? (b < 1 ? 1 : b) : 132 * 16); }

// per device: pinned slots for the running-image count of two consecutive checks
int* pinned_alive() {
    static int* h[MAX_DEVICES] = {};
    const int d = device_slot();
    if (d < 0) return nullptr;
    if (!h[d] && cudaHostAlloc((void**)&h[d], 2 * sizeof(int), cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); h[d] = nullptr; }
    return h[d];
}

}  // namespace

size_t ws_bytes_cp2(size_t M, size_t N, int batch, size_t elem) {
    const size_t n = M * N * (size_t)batch;
    return 6 * align256(n * elem) + align256((size_t)batch * sizeof(int)) + align256(3 * (size_t)batch * SLOTS * 2 * sizeof(double)) + 256;
}

template <typename T>
cudaError_t cp2_device(size_t M, size_t N, int batch, int row_major, const T* Y, double lambda, bool weighted, const T* W1, const T* W2,
                       T* out, int alg, int maxit, int* iters, void* ws, cudaStream_t st, void* tape) {
    Geom g;
    g.F = (int)(row_major ? N : M); g.S = (int)(row_major ? M : N);
    g.img = (long long)M * (long long)N; g.batch = batch;
    g.ntf = (g.F + TF - 1) / TF; g.tiles = g.ntf * ((g.S + TS - 1) / TS);
    const long long n = g.img * batch;
    char* w = (char*)ws;
    T* Xb[2]; T* Ufb[2]; T* Usb[2];
    for (int i = 0; i < 2; i++) { Xb[i] = (T*)w; w += align256(n * sizeof(T)); }
    for (int i = 0; i < 2; i++) { Ufb[i] = (T*)w; w += align256(n * sizeof(T)); }
    for (int i = 0; i < 2; i++) { Usb[i] = (T*)w; w += align256(n * sizeof(T)); }
    int* stopped = (int*)w; w += align256((size_t)batch * sizeof(int));
    double* sums = (double*)w; w += align256(3 * (size_t)batch * SLOTS * 2 * sizeof(double));
    int* d_alive = (int*)w;
    const T* Wf = row_major ? W2 : W1;
    const T* Ws = row_major ? W1 : W2;
    int* h_alive = pinned_alive();
    if (!h_alive) return cudaErrorMemoryAllocation;
    cudaEvent_t ev[2];
    for (int i = 0; i < 2; i++) {
        cudaError_t e = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming);
        if (e != cudaSuccess) { if (i) cudaEventDestroy(ev[0]); return e; }
    }
    cudaError_t err = cudaSuccess;
#define CP2_TRY(expr) do { err = (expr); if (err != cudaSuccess) goto done; } while (0)
    {
        if (maxit <= 0) maxit = 2500;                                             // MAX_ITERS_CONDAT, src/TVopt.h:75
        double sigma = 10, tau = .9 / (sigma * 8), theta = 1., gamma = alg == 2 ? 1. / lambda : 0.;
        CP2_TRY(cudaMemsetAsync(stopped, 0, (size_t)batch * sizeof(int), st));
        CP2_TRY(cudaMemsetAsync(sums, 0, 3 * (size_t)batch * SLOTS * 2 * sizeof(double), st));
        k_cp2_init<T><<<grid_1d(n), 256, 0, st>>>(g, Y, Xb[0], Ufb[0], Usb[0]);
        CP2_TRY(cudaGetLastError());
        const dim3 grid((unsigned)g.tiles, (unsigned)(batch < 65535 ? batch : 65535));
        int it = 1, pending = -1;                 // pending: the chunk whose running-image count has not been read yet
        for (int chunk = 0; it <= maxit; chunk++) {
            const int last = it + ITERS_PER_CHECK - 1 < maxit ? it + ITERS_PER_CHECK - 1 : maxit;
            for (; it <= last; it++) {
                const double cc = 1. / (1. + tau), tau_i = tau, theta_i = theta;
                if (alg == 2) { tau *= theta; sigma /= theta; theta = 1. / sqrt(1 + 2 * gamma * tau); }
                const int r = (it - 1) & 1, wr = it & 1;
                if (weighted)
                    k_cp2_iter<T, true><<<grid, THREADS, 0, st>>>(g, Y, Xb[r], Ufb[r], Usb[r], Xb[wr], Ufb[wr], Usb[wr], stopped, sums, it, alg,
                                                                  (T)tau_i, (T)cc, (T)theta_i, (T)sigma, T(0), Wf, Ws);
                else
                    k_cp2_iter<T, false><<<grid, THREADS, 0, st>>>(g, Y, Xb[r], Ufb[r], Usb[r], Xb[wr], Ufb[wr], Usb[wr], stopped, sums, it, alg,
                                                                   (T)tau_i, (T)cc, (T)theta_i, (T)sigma, (T)lambda, nullptr, nullptr);
                CP2_TRY(cudaGetLastError());
            }
            if (it > maxit) break;
            // read the count of the previous chunk while this one runs: the queue keeps at most one chunk of launches past the end
            k_cp2_alive<<<1, 256, 0, st>>>(stopped, sums, batch, it - 1, d_alive + (chunk & 1));
            CP2_TRY(cudaGetLastError());
            CP2_TRY(cudaMemcpyAsync(h_alive + (chunk & 1), d_alive + (chunk & 1), sizeof(int), cudaMemcpyDeviceToHost, st));
            CP2_TRY(cudaEventRecord(ev[chunk & 1], st));
            if (pending >= 0) {
                CP2_TRY(cudaEventSynchronize(ev[pending & 1]));
                if (h_alive[pending & 1] == 0) break;
            }
            pending = chunk;
        }
        k_cp2_out<T><<<grid_1d(n), 256, 0, st>>>(g, Xb[0], Xb[1], stopped, it, out);
        CP2_TRY(cudaGetLastError());
        if (tape) CP2_TRY(cp2_tape_tail<T>(M, N, batch, row_major, out, Ufb, Usb, stopped, it, lambda, weighted, Wf, Ws, tape, st));
        if (iters) {
            CP2_TRY(cudaMemcpyAsync(iters, stopped, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost, st));
            CP2_TRY(cudaStreamSynchronize(st));
            for (int b = 0; b < batch; b++) if (!iters[b]) iters[b] = it;
        }
    }
#undef CP2_TRY
done:
    cudaEventDestroy(ev[0]); cudaEventDestroy(ev[1]);
    return err;
}

template cudaError_t cp2_device<double>(size_t, size_t, int, int, const double*, double, bool, const double*, const double*, double*, int,
                                        int, int*, void*, cudaStream_t, void*);
template cudaError_t cp2_device<float>(size_t, size_t, int, int, const float*, double, bool, const float*, const float*, float*, int, int,
                                       int*, void*, cudaStream_t, void*);

}  // namespace ptv
