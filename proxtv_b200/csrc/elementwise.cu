// elementwise.cu -- streaming helpers of the outer loops (unfused forms; the chunked kernels fuse most of these).
//
// Arithmetic is written in the reference's operation order so that, given identical prox outputs, every intermediate is
// bit-identical to the reference's (src/TV2Dopt.cpp:390-430, :212-277; src/TVNDopt.cpp:212-227).  The only exception is
// the two sums (image mean, stop criterion), which are tree reductions with a fixed, deterministic order instead of the
// reference's serial / OpenMP-reduction order.
#include "ptv_internal.h"
#include <stdint.h>

namespace ptv {

static inline unsigned grid_for(long long n, int threads, int per_thread = 4) {
    long long b = (n + (long long)threads * per_thread - 1) / ((long long)threads * per_thread);
    if (b < 1) b = 1;
    if (b > 132LL * 32) b = 132LL * 32;         // grid-stride loops: 32 blocks per SM of an H100 (132 SMs)
    return (unsigned)b;
}

__device__ __forceinline__ double block_sum(double v) {
    __shared__ double sm[32];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) sm[w] = v;
    __syncthreads();
    int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? sm[threadIdx.x] : 0.0;
    if (w == 0) for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    return v;   // valid in thread 0
}

// ---- per-image 2*mean (DR initialisation, src/TV2Dopt.cpp:390-395) ----
template <typename T>
__global__ void k_image_partial(const T* __restrict__ Y, long long per_image, double* __restrict__ partial) {
    const T* img = Y + (long long)blockIdx.y * per_image;
    double acc = 0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < per_image; q += (long long)gridDim.x * blockDim.x)
        acc += (double)img[q];
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(long long)blockIdx.y * gridDim.x + blockIdx.x] = acc;
}
template <typename T>
__global__ void k_image_fill(T* __restrict__ t, long long per_image, const double* __restrict__ partial, int nblk) {
    __shared__ double mean2;
    double acc = 0;
    for (int q = threadIdx.x; q < nblk; q += blockDim.x) acc += partial[(long long)blockIdx.y * nblk + q];
    acc = block_sum(acc);
    if (threadIdx.x == 0) mean2 = 2 * acc / (double)per_image;
    __syncthreads();
    T v = (T)mean2;
    T* img = t + (long long)blockIdx.y * per_image;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < per_image; q += (long long)gridDim.x * blockDim.x)
        img[q] = v;
}
template <typename T>
cudaError_t ew_image_means_x2(const T* Y, long long per_image, int batch, T* t, double* scratch, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 2 * ((batch + 0) > 0 ? 1 : 0), st);
    int nblk = (int)grid_for(per_image, 256, 8);
    if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    // scratch holds REDUCE_BLOCKS doubles: split them between the images of one launch
    int share = REDUCE_BLOCKS / (batch < REDUCE_BLOCKS ? batch : REDUCE_BLOCKS);
    if (nblk > share) nblk = share < 1 ? 1 : share;
    int per_launch = REDUCE_BLOCKS / nblk; if (per_launch < 1) per_launch = 1;
    for (int b0 = 0; b0 < batch; b0 += per_launch) {
        int nb = batch - b0 < per_launch ? batch - b0 : per_launch;
        dim3 g(nblk, nb);
        k_image_partial<T><<<g, 256, 0, st>>>(Y + (long long)b0 * per_image, per_image, scratch);
        k_image_fill<T><<<g, 256, 0, st>>>(t + (long long)b0 * per_image, per_image, scratch, nblk);
    }
    return cudaGetLastError();
}

// ---- Douglas-Rachford elementwise steps ----
template <typename T> __global__ void k_dr_reflect_cols(const T* __restrict__ t, const T* __restrict__ x, T* __restrict__ s, long long n) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        T d = t[q] - x[q];                 // DR_proxDiff: in - prox(in)            (:545-546)
        s[q] = T(2) * d - t[q];            // reflection                            (:411)
    }
}
template <typename T> __global__ void k_dr_combine_rows(const T* __restrict__ Y, const T* __restrict__ s, const T* __restrict__ x,
                                                       T* __restrict__ t, long long n) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        T in = Y[q] - s[q];                // :515
        T tb = Y[q] - (in - x[q]);         // :520 with :546
        tb = T(2) * tb - s[q];             // :419
        t[q] = T(0.5) * (t[q] + tb);       // :422
    }
}
template <typename T> __global__ void k_dr_final_cols(const T* __restrict__ t, const T* __restrict__ x, T* __restrict__ s, long long n) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
        s[q] = t[q] - x[q];                // :427
}
template <typename T> __global__ void k_dr_final_rows(const T* __restrict__ Y, const T* __restrict__ s, const T* __restrict__ x,
                                                     T* __restrict__ out, long long n) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        T in = Y[q] - s[q];
        T tb = Y[q] - (in - x[q]);         // :429
        out[q] = tb - s[q];                // :430
    }
}
template <typename T> __global__ void k_dual_update(T* __restrict__ p, const T* __restrict__ a, const T* __restrict__ b, long long n) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
        p[q] += a[q] - b[q];               // src/TV2Dopt.cpp:213,:263
}

template <typename T> cudaError_t ew_dr_reflect_cols(const T* t, const T* x, T* s, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dr_reflect_cols<T><<<grid_for(n, 256), 256, 0, st>>>(t, x, s, n); return cudaGetLastError(); }
template <typename T> cudaError_t ew_dr_combine_rows(const T* Y, const T* s, const T* x, T* t, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dr_combine_rows<T><<<grid_for(n, 256), 256, 0, st>>>(Y, s, x, t, n); return cudaGetLastError(); }
template <typename T> cudaError_t ew_dr_final_cols(const T* t, const T* x, T* s, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dr_final_cols<T><<<grid_for(n, 256), 256, 0, st>>>(t, x, s, n); return cudaGetLastError(); }
template <typename T> cudaError_t ew_dr_final_rows(const T* Y, const T* s, const T* x, T* out, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dr_final_rows<T><<<grid_for(n, 256), 256, 0, st>>>(Y, s, x, out, n); return cudaGetLastError(); }
template <typename T> cudaError_t ew_dual_update(T* p, const T* a, const T* b, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dual_update<T><<<grid_for(n, 256), 256, 0, st>>>(p, a, b, n); return cudaGetLastError(); }

// ---- first DR pass on a constant image: s = 2 (t - x1[image][k]) - t, k = position of the sample along its axis-0 fiber ----
template <typename T> __global__ void k_dr_reflect_bcast(const T* __restrict__ t, const T* __restrict__ x1, T* __restrict__ s, long long n,
                                                        long long per_image, int len, long long inc) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const long long b = q / per_image, r = q - b * per_image;
        const int k = (int)((r / inc) % len);
        const T d = t[q] - x1[b * len + k];
        s[q] = T(2) * d - t[q];
    }
}
template <typename T> cudaError_t ew_dr_reflect_bcast(const T* t, const T* x1, T* s, long long n, long long per_image, int len,
                                                      long long inc, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    k_dr_reflect_bcast<T><<<grid_for(n, 256), 256, 0, st>>>(t, x1, s, n, per_image, len, inc); return cudaGetLastError(); }

// sums the nblk partials of one reduction in a fixed order: *result = that / n
__global__ void k_final_mean(const double* __restrict__ partial, int nblk, long long n, double* __restrict__ result) {
    double acc = 0;
    for (int q = threadIdx.x; q < nblk; q += blockDim.x) acc += partial[q];
    acc = block_sum(acc);
    if (threadIdx.x == 0) *result = acc / (double)n;
}

// ---- the proximal Dykstra solvers' combine and stop value (PD_TV / PD2_TV, src/TVNDopt.cpp:212-227, src/TV2Dopt.cpp:273-277), for
//      `items` running items at once (DESIGN.md section 16; a single-item call is one item) ----
// A 2D grid: blockIdx.y = slot s0 + y of the running items, each item n elements at s * n; blockIdx.x = one of the nblk reduction blocks
// an item of n elements gets.  The element-to-thread assignment inside an item goes by element index, not address, so an item sums in
// the same order in every slot and in every batch.  partial[s * nblk + x].
constexpr int MAX_GRID_Y = 65535;

// PD_TV's combine, x = sum_i p_i/k ; z_i += x - p_i ; stop = mean|x - x_old|.  k_pd_combine_items: K 1..4 known at compile time, the 2K
// array pointers passed by value, V = 16 / sizeof(T) consecutive elements per thread step, the trailing n % V by block 0's thread 0
// after its loop; VLD: every item's arrays are 16-byte aligned, so the V elements move as one vector.  k_pd_combine_items_gen: any k,
// one element per step, the pointer tables in device memory.
template <typename T, int K> struct PdPtrs { T* p[K]; T* z[K]; };
template <typename T>
__global__ void k_pd_combine_items_gen(T* const* __restrict__ p, T* const* __restrict__ z, int k, T* __restrict__ x, long long n, int s0,
                                       double* __restrict__ partial) {
    const long long base = (long long)(s0 + blockIdx.y) * n;
    double acc = 0;
    const T kk = (T)k;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const long long e = base + q;
        T xo = x[e], xn = T(0);
        for (int i = 0; i < k; i++) xn += p[i][e] / kk;
        for (int i = 0; i < k; i++) z[i][e] += xn - p[i][e];
        x[e] = xn;
        acc += fabs((double)xn - (double)xo);
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(long long)(s0 + blockIdx.y) * gridDim.x + blockIdx.x] = acc;
}
template <typename T, int K, bool VLD>
__global__ void __launch_bounds__(256, 1) k_pd_combine_items(PdPtrs<T, K> a, T* __restrict__ x, long long n, int s0, double* __restrict__ partial) {
    const long long base = (long long)(s0 + blockIdx.y) * n;
    double acc = 0;
    {
        constexpr int V = 16 / (int)sizeof(T);
        struct alignas(16) Vec { T v[V]; };
        const T kk = (T)K;
        const long long nv = n / V;
        for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nv; q += (long long)gridDim.x * blockDim.x) {
            const long long e0 = base + q * V;
            T xo[V], pv[K][V], zv[K][V], xn[V];
            if constexpr (VLD) {
                const Vec a0 = *reinterpret_cast<const Vec*>(x + e0);
#pragma unroll
                for (int c = 0; c < V; c++) xo[c] = a0.v[c];
#pragma unroll
                for (int i = 0; i < K; i++) {
                    const Vec a1 = *reinterpret_cast<const Vec*>(a.p[i] + e0), a2 = *reinterpret_cast<const Vec*>(a.z[i] + e0);
#pragma unroll
                    for (int c = 0; c < V; c++) { pv[i][c] = a1.v[c]; zv[i][c] = a2.v[c]; }
                }
            } else {
#pragma unroll
                for (int c = 0; c < V; c++) {
                    xo[c] = x[e0 + c];
#pragma unroll
                    for (int i = 0; i < K; i++) { pv[i][c] = a.p[i][e0 + c]; zv[i][c] = a.z[i][e0 + c]; }
                }
            }
#pragma unroll
            for (int c = 0; c < V; c++) {
                T s = T(0);
#pragma unroll
                for (int i = 0; i < K; i++) s += pv[i][c] / kk;
#pragma unroll
                for (int i = 0; i < K; i++) zv[i][c] += s - pv[i][c];
                xn[c] = s;
                acc += fabs((double)s - (double)xo[c]);
            }
            if constexpr (VLD) {
#pragma unroll
                for (int i = 0; i < K; i++) {
                    Vec o;
#pragma unroll
                    for (int c = 0; c < V; c++) o.v[c] = zv[i][c];
                    *reinterpret_cast<Vec*>(a.z[i] + e0) = o;
                }
                Vec o;
#pragma unroll
                for (int c = 0; c < V; c++) o.v[c] = xn[c];
                *reinterpret_cast<Vec*>(x + e0) = o;
            } else {
#pragma unroll
                for (int c = 0; c < V; c++) {
#pragma unroll
                    for (int i = 0; i < K; i++) a.z[i][e0 + c] = zv[i][c];
                    x[e0 + c] = xn[c];
                }
            }
        }
        if (blockIdx.x == 0 && threadIdx.x == 0)                   // the < V trailing elements of the item
            for (long long e = base + nv * V; e < base + n; e++) {
                T xo = x[e], s = T(0);
                for (int i = 0; i < K; i++) s += a.p[i][e] / kk;
                for (int i = 0; i < K; i++) a.z[i][e] += s - a.p[i][e];
                x[e] = s; acc += fabs((double)s - (double)xo);
            }
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(long long)(s0 + blockIdx.y) * gridDim.x + blockIdx.x] = acc;
}
// PD2_TV's stop value, mean |a - b|
template <typename T> __global__ void k_absdiff_items(const T* __restrict__ a, const T* __restrict__ b, long long n, int s0,
                                                      double* __restrict__ partial) {
    const long long base = (long long)(s0 + blockIdx.y) * n;
    double acc = 0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
        acc += fabs((double)a[base + q] - (double)b[base + q]);
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(long long)(s0 + blockIdx.y) * gridDim.x + blockIdx.x] = acc;
}
// k_final_mean per item: block s sums its nblk partials, result[s] = that / n
__global__ void k_final_mean_items(const double* __restrict__ partial, int nblk, long long n, double* __restrict__ result) {
    double acc = 0;
    for (int q = threadIdx.x; q < nblk; q += blockDim.x) acc += partial[(long long)blockIdx.x * nblk + q];
    acc = block_sum(acc);
    if (threadIdx.x == 0) result[blockIdx.x] = acc / (double)n;
}

template <typename T, int K>
static void launch_pd_items(T* const* hp, T* const* hz, bool vld, T* x, long long n, int s0, int ny, double* scratch, int nblk, cudaStream_t st) {
    PdPtrs<T, K> a;
    for (int i = 0; i < K; i++) { a.p[i] = hp[i]; a.z[i] = hz[i]; }
    if (vld) k_pd_combine_items<T, K, true><<<dim3(nblk, ny), 256, 0, st>>>(a, x, n, s0, scratch);
    else k_pd_combine_items<T, K, false><<<dim3(nblk, ny), 256, 0, st>>>(a, x, n, s0, scratch);
}
// dp, dz: device copies of the pointer arrays (generic kernel); hp, hz: the same pointers on the host (K <= 4)
template <typename T> cudaError_t ew_pd_combine_items(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                      int items, double* scratch, double* result, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1 + (items + MAX_GRID_Y - 1) / MAX_GRID_Y, st);
    // the vector assignment for 1..4 terms when x and every p_i / z_i are 16-byte aligned (a batch's arrays are workspace, so always);
    // VLD when every slot is aligned too: n * sizeof(T) a multiple of 16, or slot 0 alone
    bool vec = k >= 1 && k <= 4 && (((uintptr_t)x) & 15) == 0;
    for (int i = 0; i < k && vec; i++) vec = ((((uintptr_t)hp[i]) | ((uintptr_t)hz[i])) & 15) == 0;
    const bool vld = items == 1 || ((n * (long long)sizeof(T)) & 15) == 0;
    int nblk = vec ? (int)grid_for(n, 256, 16 / (int)sizeof(T) * 2) : (int)grid_for(n, 256, 4);
    if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    for (int s0 = 0; s0 < items; s0 += MAX_GRID_Y) {
        const int ny = items - s0 < MAX_GRID_Y ? items - s0 : MAX_GRID_Y;
        switch (vec ? k : 0) {
            case 1: launch_pd_items<T, 1>(hp, hz, vld, x, n, s0, ny, scratch, nblk, st); break;
            case 2: launch_pd_items<T, 2>(hp, hz, vld, x, n, s0, ny, scratch, nblk, st); break;
            case 3: launch_pd_items<T, 3>(hp, hz, vld, x, n, s0, ny, scratch, nblk, st); break;
            case 4: launch_pd_items<T, 4>(hp, hz, vld, x, n, s0, ny, scratch, nblk, st); break;
            default: k_pd_combine_items_gen<T><<<dim3(nblk, ny), 256, 0, st>>>(dp, dz, k, x, n, s0, scratch); break;
        }
    }
    k_final_mean_items<<<items, 256, 0, st>>>(scratch, nblk, n, result);
    return cudaGetLastError();
}
template <typename T> cudaError_t ew_mean_abs_diff_items(const T* a, const T* b, long long n, int items, double* scratch, double* result,
                                                         cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1 + (items + MAX_GRID_Y - 1) / MAX_GRID_Y, st);
    int nblk = (int)grid_for(n, 256, 8); if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    for (int s0 = 0; s0 < items; s0 += MAX_GRID_Y) {
        const int ny = items - s0 < MAX_GRID_Y ? items - s0 : MAX_GRID_Y;
        k_absdiff_items<T><<<dim3(nblk, ny), 256, 0, st>>>(a, b, n, s0, scratch);
    }
    k_final_mean_items<<<items, 256, 0, st>>>(scratch, nblk, n, result);
    return cudaGetLastError();
}

// Moves whole n-element slots: dst slot s = src slot map[s] when map[s] >= 0; map[s] = -1 - b: item b joins, with the start value init
// 0: 0 ; 1: G_b / kk ; 2: G_b / kk - 0 ; 3: G_b - 0 (G_b = G + b n, the start values of the PD_TV / PD2_TV backward, dr2_vjp.cu).
// src is not read when every map[s] < 0.
template <typename T> __global__ void k_slot_gather(const T* __restrict__ src, T* __restrict__ dst, const int* __restrict__ map, long long n,
                                                    int slots, int init, const T* __restrict__ G, T kk) {
    for (int s = blockIdx.y; s < slots; s += gridDim.y) {          // slots along y: no division per element
        const int m = map[s];
        T* d = dst + (long long)s * n;
        for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
            if (m >= 0) { d[e] = src[(long long)m * n + e]; continue; }
            const T g = init ? G[(long long)(-1 - m) * n + e] : T(0);
            d[e] = init == 0 ? T(0) : init == 1 ? g / kk : init == 2 ? g / kk - T(0) : g - T(0);
        }
    }
}
template <typename T> cudaError_t ew_slot_gather(const T* src, T* dst, const int* map, int slots, long long n, int init, const T* G, T kk,
                                                 cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    const unsigned gx = grid_for(n, 256);
    unsigned gy = 132u * 32 / gx;                                   // grid_for's block budget, shared by the slots
    if (gy > (unsigned)slots) gy = (unsigned)slots;
    if (gy > (unsigned)MAX_GRID_Y) gy = MAX_GRID_Y;
    if (gy < 1) gy = 1;
    k_slot_gather<T><<<dim3(gx, gy), 256, 0, st>>>(src, dst, map, n, slots, init, G, kk);
    return cudaGetLastError();
}

// ---- parallel Douglas-Rachford combine (src/TVNDopt.cpp:456-475): q = sum_i p_i/k ; x = sum_i z_i/k (both accumulated term by
//      term) ; z_i += 2 q - x - p_i ; stop = mean|x - x_old| ----
template <typename T> __global__ void k_pdr_combine(T* const* __restrict__ p, T* const* __restrict__ z, int k, T* __restrict__ x,
                                                   long long n, double* __restrict__ partial) {
    double acc = 0;
    const T kk = (T)k;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        T xo = x[e], xn = T(0), q = T(0);
        for (int i = 0; i < k; i++) { q += p[i][e] / kk; xn += z[i][e] / kk; }
        for (int i = 0; i < k; i++) z[i][e] += T(2) * q - xn - p[i][e];
        x[e] = xn;
        acc += fabs((double)xn - (double)xo);
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}
template <typename T, int K>
__global__ void __launch_bounds__(256) k_pdr_combine_vec(PdPtrs<T, K> a, T* __restrict__ x, long long n, double* __restrict__ partial) {
    constexpr int V = 16 / (int)sizeof(T);
    struct alignas(16) Vec { T v[V]; };
    double acc = 0;
    const T kk = (T)K;
    const long long nv = n / V;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < nv; e += (long long)gridDim.x * blockDim.x) {
        Vec xo = reinterpret_cast<const Vec*>(x)[e], pv[K], zv[K], xn;
#pragma unroll
        for (int i = 0; i < K; i++) { pv[i] = reinterpret_cast<const Vec*>(a.p[i])[e]; zv[i] = reinterpret_cast<const Vec*>(a.z[i])[e]; }
#pragma unroll
        for (int c = 0; c < V; c++) {
            T q = T(0), s = T(0);
#pragma unroll
            for (int i = 0; i < K; i++) { q += pv[i].v[c] / kk; s += zv[i].v[c] / kk; }
#pragma unroll
            for (int i = 0; i < K; i++) zv[i].v[c] += T(2) * q - s - pv[i].v[c];
            xn.v[c] = s;
            acc += fabs((double)s - (double)xo.v[c]);
        }
#pragma unroll
        for (int i = 0; i < K; i++) reinterpret_cast<Vec*>(a.z[i])[e] = zv[i];
        reinterpret_cast<Vec*>(x)[e] = xn;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0)                       // the < V trailing elements
        for (long long e = nv * V; e < n; e++) {
            T xo = x[e], s = T(0), q = T(0);
            for (int i = 0; i < K; i++) { q += a.p[i][e] / kk; s += a.z[i][e] / kk; }
            for (int i = 0; i < K; i++) a.z[i][e] += T(2) * q - s - a.p[i][e];
            x[e] = s; acc += fabs((double)s - (double)xo);
        }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}
template <typename T, int K>
static void launch_pdr_vec(T* const* hp, T* const* hz, T* x, long long n, double* scratch, int nblk, cudaStream_t st) {
    PdPtrs<T, K> a;
    for (int i = 0; i < K; i++) { a.p[i] = hp[i]; a.z[i] = hz[i]; }
    k_pdr_combine_vec<T, K><<<nblk, 256, 0, st>>>(a, x, n, scratch);
}
template <typename T> cudaError_t ew_pdr_combine(T* const* dp, T* const* dz, T* const* hp, T* const* hz, int k, T* x, long long n,
                                                 double* scratch, double* result, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 2, st);
    bool aligned = (((uintptr_t)x) & 15) == 0;
    for (int i = 0; i < k && aligned; i++) aligned = ((((uintptr_t)hp[i]) | ((uintptr_t)hz[i])) & 15) == 0;
    int nblk;
    if (aligned && k >= 1 && k <= 4) {
        nblk = (int)grid_for(n, 256, 16 / (int)sizeof(T) * 2); if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
        switch (k) {
            case 1: launch_pdr_vec<T, 1>(hp, hz, x, n, scratch, nblk, st); break;
            case 2: launch_pdr_vec<T, 2>(hp, hz, x, n, scratch, nblk, st); break;
            case 3: launch_pdr_vec<T, 3>(hp, hz, x, n, scratch, nblk, st); break;
            default: launch_pdr_vec<T, 4>(hp, hz, x, n, scratch, nblk, st); break;
        }
    } else {
        nblk = (int)grid_for(n, 256, 4); if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
        k_pdr_combine<T><<<nblk, 256, 0, st>>>(dp, dz, k, x, n, scratch);
    }
    k_final_mean<<<1, 256, 0, st>>>(scratch, nblk, n, result);
    return cudaGetLastError();
}
// x = y / k (src/TVNDopt.cpp:367)
template <typename T> __global__ void k_div_scalar(const T* __restrict__ y, T* __restrict__ x, long long n, T kk) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) x[e] = y[e] / kk;
}
template <typename T> cudaError_t ew_div_scalar(const T* y, T* x, long long n, T k, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    int nblk = (int)grid_for(n, 256, 8); if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    k_div_scalar<T><<<nblk, 256, 0, st>>>(y, x, n, k);
    return cudaGetLastError();
}

// first Douglas-Rachford half-iteration on the constant start image t (2 * mean): the column prox of a constant is that constant, so
// d = t - x_cols and u = Y - (2 d - t) need no scan; written with the very expressions the lane drain uses (PassOp<LOP_DRA>)
template <typename T> __global__ void k_dr_first(const T* Y, const T* __restrict__ t, T* __restrict__ U, T* D, long long n) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const T c = t[e], d = c - c, y = Y[e];            // Y may be D (in place): read before the write
        D[e] = d; U[e] = y - (T(2) * d - c);
    }
}
template <typename T> cudaError_t ew_dr_first(const T* Y, const T* t, T* U, T* D, long long n, cudaStream_t st) {
    KernelSpan span(KC_ELEMENTWISE, 1, st);
    int nblk = (int)grid_for(n, 256, 8); if (nblk > REDUCE_BLOCKS) nblk = REDUCE_BLOCKS;
    k_dr_first<T><<<nblk, 256, 0, st>>>(Y, t, U, D, n);
    return cudaGetLastError();
}

// mean |y[e + 1] - y[e]| over n consecutive elements (the lane-engine suitability test, solver.cu), in a fixed summation order: the
// terms of e = j, j + 256, j + 512, ... are summed in that order into s_j, and the 256 sums s_j are combined by a pairwise tree.
// Block j of k_abs_step_lanes forms s_j: its 256 threads load the terms (all loads in flight at once) into shared memory, one thread
// adds them up; the serial chain is then shared-memory adds only, not one dependent global round trip per term as in a single block
// of 256 threads walking the array (~400 us for 256k float64 elements on an H100, on every call of a solver under engine auto).
constexpr int ABS_STEP_LANES = 256, ABS_STEP_CHUNK = 1024;
template <typename T> __global__ void __launch_bounds__(256) k_abs_step_lanes(const T* __restrict__ y, long long n, double* __restrict__ part) {
    __shared__ double term[ABS_STEP_CHUNK];
    const long long j = blockIdx.x;
    const long long cnt = n - 1 > j ? (n - 2 - j) / ABS_STEP_LANES + 1 : 0;          // e = j + k 256 with e + 1 < n
    double s = 0.0;
    for (long long k0 = 0; k0 < cnt; k0 += ABS_STEP_CHUNK) {
        const int m = cnt - k0 < ABS_STEP_CHUNK ? (int)(cnt - k0) : ABS_STEP_CHUNK;
        for (int k = threadIdx.x; k < m; k += blockDim.x) {
            const long long e = j + (k0 + k) * ABS_STEP_LANES;
            term[k] = fabs((double)y[e + 1] - (double)y[e]);
        }
        __syncthreads();
        if (threadIdx.x == 0)
            for (int k = 0; k < m; k++) s += term[k];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[j] = s;
}
__global__ void k_abs_step_tree(const double* __restrict__ part, long long n, double* __restrict__ out) {
    __shared__ double sh[ABS_STEP_LANES];
    sh[threadIdx.x] = part[threadIdx.x];
    __syncthreads();
    for (int k = ABS_STEP_LANES / 2; k > 0; k >>= 1) { if ((int)threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k]; __syncthreads(); }
    if (threadIdx.x == 0) out[0] = n > 1 ? sh[0] / (double)(n - 1) : 0.0;
}
template <typename T> cudaError_t ew_mean_abs_step(const T* y, long long n, double* out, cudaStream_t st) {
    k_abs_step_lanes<T><<<ABS_STEP_LANES, 256, 0, st>>>(y, n, out + 1);
    k_abs_step_tree<<<1, ABS_STEP_LANES, 0, st>>>(out + 1, n, out);
    return cudaGetLastError();
}

#define INST(T) \
    template cudaError_t ew_mean_abs_step<T>(const T*, long long, double*, cudaStream_t); \
    template cudaError_t ew_dr_first<T>(const T*, const T*, T*, T*, long long, cudaStream_t); \
    template cudaError_t ew_image_means_x2<T>(const T*, long long, int, T*, double*, cudaStream_t); \
    template cudaError_t ew_dr_reflect_cols<T>(const T*, const T*, T*, long long, cudaStream_t); \
    template cudaError_t ew_dr_combine_rows<T>(const T*, const T*, const T*, T*, long long, cudaStream_t); \
    template cudaError_t ew_dr_final_cols<T>(const T*, const T*, T*, long long, cudaStream_t); \
    template cudaError_t ew_dr_final_rows<T>(const T*, const T*, const T*, T*, long long, cudaStream_t); \
    template cudaError_t ew_dual_update<T>(T*, const T*, const T*, long long, cudaStream_t); \
    template cudaError_t ew_dr_reflect_bcast<T>(const T*, const T*, T*, long long, long long, int, long long, cudaStream_t); \
    template cudaError_t ew_pdr_combine<T>(T* const*, T* const*, T* const*, T* const*, int, T*, long long, double*, double*, cudaStream_t); \
    template cudaError_t ew_pd_combine_items<T>(T* const*, T* const*, T* const*, T* const*, int, T*, long long, int, double*, double*, cudaStream_t); \
    template cudaError_t ew_mean_abs_diff_items<T>(const T*, const T*, long long, int, double*, double*, cudaStream_t); \
    template cudaError_t ew_slot_gather<T>(const T*, T*, const int*, int, long long, int, const T*, T, cudaStream_t); \
    template cudaError_t ew_div_scalar<T>(const T*, T*, long long, T, cudaStream_t);
INST(double)
INST(float)

}  // namespace ptv
