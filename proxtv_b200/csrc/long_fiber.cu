// long_fiber.cu -- contiguous fibers too long for shared memory (e.g. tv1_1d on 1e6 samples, BASELINE config 1).
//
// The fiber is cut into overlapping tiles of W = TL + HL + HR samples; every tile is solved as a stand-alone signal by the
// chunked kernel (its first / last tile own the true ends), and tile k keeps only its owned range [k TL, (k+1) TL).  The
// stand-alone solve of a tile differs from the global one only near the tile's artificial ends: the scan forgets its start
// after the first shared break (renewal states, chunk_core.cuh), and the artificial end can only re-shape the segments that
// are still open when the scan reaches it.  Two neighbouring tiles therefore agree bit for bit on the middle of their
// overlap, and if they do -- and that window contains a jump, i.e. a break both scans passed through -- the concatenation
// satisfies the optimality conditions of the whole fiber and equals the sequential scan.  That agreement is CHECKED on the
// device for every tile boundary; any failure (a segment longer than the margins) makes the caller fall back to the
// sequential kernel for the whole call, so the result is exact either way.
#include "ptv_internal.h"
#include "chunk_core.cuh"

namespace ptv {

template <typename T>
cudaError_t prox_fibers_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                       const T* lamv, cudaStream_t st, T* X2 = nullptr, long long inc2 = 0,
                                       const T* lamf = nullptr, long long fpi = 1);

constexpr int LF_TL = 8192, LF_HL = 512, LF_HR = 512, LF_W = LF_TL + LF_HL + LF_HR;

__host__ __device__ inline long long lf_tile_start(long long k, long long n) {
    long long s = k * LF_TL - LF_HL;
    if (s < 0) s = 0;
    if (s > n - LF_W) s = n - LF_W;
    return s;
}

template <typename T>
__global__ void k_lf_gather(const T* __restrict__ A, const T* __restrict__ B, int op, T* __restrict__ tiles, long long n, int nt) {
    const long long tile = blockIdx.y;                 // fiber * nt + k
    const long long f = tile / nt, k = tile % nt;
    const long long s = lf_tile_start(k, n);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < LF_W; e += gridDim.x * blockDim.x) {
        const long long g = f * n + s + e;
        T a = A[g];
        if (op == IN_A_MINUS_B) a = a - B[g]; else if (op == IN_A_PLUS_B) a = a + B[g];
        tiles[tile * LF_W + e] = a;
    }
}

// owned ranges back to the fiber + agreement check of neighbouring tiles on the middle of their overlap
template <typename T>
__global__ void k_lf_scatter_check(const T* __restrict__ sol, T* __restrict__ X, long long n, int nt, int* __restrict__ bad) {
    const long long tile = blockIdx.y;
    const long long f = tile / nt, k = tile % nt;
    const long long s = lf_tile_start(k, n);
    const long long o0 = k * LF_TL, o1 = (o0 + LF_TL < n) ? o0 + LF_TL : n;
    const T* me = sol + tile * LF_W;
    for (long long i = o0 + blockIdx.x * blockDim.x + threadIdx.x; i < o1; i += (long long)gridDim.x * blockDim.x) X[f * n + i] = me[i - s];
    if (k + 1 < nt && blockIdx.x == 0) {
        // window [c0, c1) around the boundary b = (k+1) TL, inside both tiles
        const long long b = (k + 1) * LF_TL, s2 = lf_tile_start(k + 1, n);
        long long c0 = b - LF_HL / 2, c1 = b + LF_HR / 2;
        if (c0 < s2) c0 = s2;
        if (c1 > s + LF_W) c1 = s + LF_W;
        const T* nb = sol + (tile + 1) * LF_W;
        int differ = 0, jump = 0;
        for (long long i = c0 + threadIdx.x; i < c1; i += blockDim.x) {
            const T a = me[i - s], c = nb[i - s2];
            if (!(a == c)) differ = 1;
            if (i + 1 < c1 && me[i + 1 - s] != a) jump = 1;
        }
        differ = __syncthreads_or(differ); jump = __syncthreads_or(jump);
        if (threadIdx.x == 0 && (differ || !jump)) atomicOr(bad, 1);
    }
}

// scratch: at least lf_scratch_elems(g) elements + 16 bytes.  Returns cudaErrorInvalidConfiguration if not applicable, and
// cudaErrorNotReady if the tiles did not agree (nothing valid was written: the caller must use the sequential kernel).
template <typename T>
cudaError_t prox_long_fibers(const T* A, const T* B, InOp op, T* X, int out_op, FiberGeom g, T lam, T* scratch, long long scratch_elems,
                             cudaStream_t st) {
    const long long n = g.len;
    if (g.inc != 1 || n < 2LL * LF_W || out_op > OUT_DIFF) return cudaErrorInvalidConfiguration;
    const int nt = (int)((n + LF_TL - 1) / LF_TL);
    const long long ntiles = g.nf * nt, need = 2 * ntiles * LF_W + 8;
    if (!scratch || scratch_elems < need || ntiles > 65535) return cudaErrorInvalidConfiguration;
    T* tiles = scratch; T* sol = scratch + ntiles * LF_W; int* bad = reinterpret_cast<int*>(sol + ntiles * LF_W);
    cudaError_t e = cudaMemsetAsync(bad, 0, sizeof(int), st);
    if (e != cudaSuccess) return e;
    dim3 grid(8, (unsigned)ntiles);
    k_lf_gather<T><<<grid, 256, 0, st>>>(A, B, (int)op, tiles, n, nt);
    e = prox_fibers_chunked_contig<T>(tiles, nullptr, nullptr, IN_A, sol, out_op, FiberGeom{ntiles, LF_W, 1}, lam, nullptr, st);
    if (e != cudaSuccess) return e;
    k_lf_scatter_check<T><<<grid, 256, 0, st>>>(sol, X, n, nt, bad);
    int hbad = 0;
    e = cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return e;
    return hbad ? cudaErrorNotReady : cudaGetLastError();
}

long long lf_scratch_elems(long long nf, long long len) {
    const long long nt = (len + LF_TL - 1) / LF_TL;
    return 2 * nf * nt * LF_W + 8;
}

template cudaError_t prox_long_fibers<double>(const double*, const double*, InOp, double*, int, FiberGeom, double, double*, long long, cudaStream_t);
template cudaError_t prox_long_fibers<float>(const float*, const float*, InOp, float*, int, FiberGeom, float, float*, long long, cudaStream_t);

}  // namespace ptv
