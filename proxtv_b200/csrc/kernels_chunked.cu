// kernels_chunked.cu -- chunked speculative TV-L1 prox: many lanes per fiber, exact stitching (phases in chunk_core.cuh).
//
// k_prox_chunked_contig: contiguous fibers (element stride 1).  A CTA stages `fpb` whole fibers in shared memory
// (chunk rows padded by 16 B so lanes that walk their chunks in lock-step do not all hit one bank), runs
// walk-own-chunk -> rounds -> fill with one lane per 32-sample chunk, and streams the fused result back with coalesced
// stores.  HBM traffic per launch: every input array read once, the output written once.
#include "ptv_internal.h"
#include "chunk_core.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace ptv {

template <typename T> struct PadCfg { static constexpr int PADE = 16 / (int)sizeof(T); };   // 16 bytes of padding per chunk row

template <typename T> struct SmemLd {
    const T* p;
    PTV_HD T operator()(int j) const { return p[j + (j >> 5) * PadCfg<T>::PADE]; }
};
template <typename T> struct SmemSt {
    T* p;
    PTV_HD void operator()(int j, T v) const { p[j + (j >> 5) * PadCfg<T>::PADE] = v; }
};

// ---- TMA (bulk async copy) staging: cp.async.bulk global -> shared, completion counted on an mbarrier ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// shared-memory sample load through a 32-bit shared-window address held in a register
template <typename T> struct SmemLd32 {
    uint32_t base;
    __device__ __forceinline__ T operator()(int j) const;
};
template <> __device__ __forceinline__ double SmemLd32<double>::operator()(int j) const {
    double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(base + (((uint32_t)j + 2u * ((uint32_t)j >> 5)) << 3)) : "memory"); return v;
}
template <> __device__ __forceinline__ float SmemLd32<float>::operator()(int j) const {
    float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(base + (((uint32_t)j + 4u * ((uint32_t)j >> 5)) << 2)) : "memory"); return v;
}

// make a kernel parameter an opaque register value: stops the compiler from re-loading it from the constant bank inside the
// scan loop (each reload costs an LDC plus its latency on the dependent compare)
__device__ __forceinline__ double in_register(double v) { asm volatile("" : "+d"(v)); return v; }
__device__ __forceinline__ float in_register(float v) { asm volatile("" : "+f"(v)); return v; }
__device__ __forceinline__ int in_register(int v) { asm volatile("" : "+r"(v)); return v; }

template <typename T> struct GlobSt {            // sparse value store = the fiber's own output row (see chunk_core.cuh)
    T* p;                                        // per-lane register copy of the row pointer: one IMAD.WIDE per store
    __device__ __forceinline__ void operator()(int j, T v) const { p[(unsigned)j] = v; }
};
__device__ __forceinline__ double* in_register(double* v) { asm volatile("" : "+l"(v)); return v; }
__device__ __forceinline__ float* in_register(float* v) { asm volatile("" : "+l"(v)); return v; }

#ifdef PTV_PHASE_TIMING
// debug build only (make EXTRA=-DPTV_PHASE_TIMING): per-phase CTA time of the contiguous kernel, summed over CTAs
__device__ unsigned long long g_phase_ns[8];
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define PHASE_MARK(k) do { if (threadIdx.x == 0) { const unsigned long long t_ = gtime(); atomicAdd(&g_phase_ns[k], t_ - t_prev); t_prev = t_; } } while (0)
#else
#define PHASE_MARK(k) do { } while (0)
#endif

// One batch of the fill phase: FW consecutive 32-sample windows of one fiber, handled by one warp (see the kernel).
template <typename T, int FW, int CL, int CHT>
__device__ __forceinline__ void fill_batch(int c0, int nwin, int nchunks, int n, int lane, uint32_t below, T* __restrict__ xr, long long gb, long long x2b,
                                           const uint32_t* __restrict__ Pm, const T* __restrict__ cv, T* __restrict__ yr, int out_op,
                                           const T* __restrict__ A, const T* __restrict__ B, const T* __restrict__ C, T* __restrict__ X2,
                                           long long inc2) {
    constexpr int PADE = PadCfg<T>::PADE;
    T v[FW];
#pragma unroll
    for (int u = 0; u < FW; u++) {
        const int c = c0 + u;                                      // 32-sample window c = chunk c, or chunks 2c and 2c+1 (CHT == 16)
        v[u] = T(0);
        if (c < nwin && (c << 5) + lane < n) {
            const uint32_t pw = (CHT == 32) ? Pm[c] : (Pm[2 * c] | ((2 * c + 1 < nchunks) ? (Pm[2 * c + 1] << 16) : 0u));
            const uint32_t w = pw & below;
            v[u] = w ? __ldcg(xr + (c << 5) + high_bit(w)) : cv[(CHT == 32) ? c : 2 * c];
        }
    }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < FW; u++) {
        const int c = c0 + u, j = (c << 5) + lane;
        if (c < nwin && j < n) {
            const T o = apply_out_ex<T>(out_op, yr[j + c * PADE], v[u], A, B, C, gb + j);
            xr[j] = o;
            if (CL == 0) { if (X2) X2[x2b + (long long)j * inc2] = o; }      // scattered 8-byte stores
            else yr[j + c * PADE] = o;                                       // keep the finished row for the exchange
        }
    }
}

// CL: how the optional transposed second output X2 is produced.  0: plain 8-byte scattered stores (slow: partial-sector writes make
// L2 read-modify-write every sector); >= 1: the finished fiber rows of CL consecutive CTAs (a thread-block cluster when CL > 1)
// are exchanged through (distributed) shared memory so that fpb*CL adjacent fibers are written together as full 32-byte sectors.
// LAMF: fiber j's penalty is lamf[j / fpi] (one per group of fpi fibers), the uniform scan with that value.
template <typename T, bool WEIGHTED, int MAXT, int CL, int CHT = CH, bool LAMF = false>
__global__ void __launch_bounds__(MAXT, MAXT <= 256 ? 2 : 1) k_prox_chunked_contig(const T* __restrict__ A, const T* __restrict__ B, const T* __restrict__ C, int in_op,
                                      T* __restrict__ X, int out_op,
                                      long long nf, int n, T lam, const T* __restrict__ lamv, int lpf, int fpb, int npad, int use_tma,
                                      T* __restrict__ X2, long long inc2, uint32_t* __restrict__ Mk, T* __restrict__ Cv,
                                      const T* __restrict__ lamf, long long fpi) {
    __shared__ uint64_t mbar;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    RcpPair<T>* rcp = reinterpret_cast<RcpPair<T>*>(smem_raw);    // reciprocal table        [RCP_N]   (16-byte aligned)
    T* ys = reinterpret_cast<T*>(rcp + RCP_N);                    // staged input            [fpb][npad] (npad*sizeof(T) % 16 == 0)
    T* wsm = ys + (size_t)fpb * npad;                             // per-edge weights        [fpb][npad] (weighted only)
    // value entering each chunk [fpb][lpf]: only needed after the scan, so for small CTAs it re-uses the reciprocal table's
    // bytes (the table is dead once the last round's barrier has passed) -- the 1 KB saved buys a sixth resident CTA per SM
    const bool cval_aliased = (size_t)fpb * lpf <= 2 * RCP_N;
    T* cval_own = wsm + (WEIGHTED ? (size_t)fpb * npad : 0);
    T* cval = cval_aliased ? reinterpret_cast<T*>(rcp) : cval_own;
    uint32_t* mk = reinterpret_cast<uint32_t*>(cval_own + (cval_aliased ? 0 : (size_t)fpb * lpf));      // masks P, K0, K1 [3][fpb][lpf]
    constexpr int PADE = PadCfg<T>::PADE;
    const int tid = threadIdx.x;
    const long long f0 = (long long)blockIdx.x * fpb;
    const int nfib = (int)((nf - f0) < fpb ? (nf - f0) : fpb);
    const int nchunks = (n + CHT - 1) / CHT;                     // lanes per fiber
    const int nwin = (n + CH - 1) / CH;                          // 32-sample rows of the staged fiber == windows of the fill

#ifdef PTV_PHASE_TIMING
    unsigned long long t_prev = gtime();
#endif
    // ---- stage the fibers ----
    if (tid < RCP_N) { rcp[tid].r = tid ? T(1) / T(tid) : T(0); rcp[tid].d = T(tid); }
    if (use_tma) {
        // one bulk copy per 32-sample chunk row (rows are padded in shared memory), all in flight at once
        if (tid == 0) mbar_init(&mbar, 1);
        __syncthreads();
        if (tid == 0) mbar_arrive_expect_tx(&mbar, (uint32_t)((size_t)nfib * n * sizeof(T)));
        for (int e = tid; e < nfib * nwin; e += blockDim.x) {
            const int fb = e / nwin, c = e - fb * nwin;
            const int cnt = (c * CH + CH <= n) ? CH : n - c * CH;
            tma_bulk_g2s(ys + (size_t)fb * npad + (size_t)c * (CH + PADE), A + (f0 + fb) * (long long)n + (long long)c * CH,
                         (uint32_t)(cnt * sizeof(T)), &mbar);
        }
    }
    for (int fb = 0; fb < nfib; fb++) {
        const long long base = (f0 + fb) * (long long)n;
        T* row = ys + (size_t)fb * npad;
        if (!use_tma) for (int j = tid; j < n; j += blockDim.x) {       // coalesced reads, input op applied on the fly
            T a = A[base + j];
            if (in_op == IN_A_MINUS_B) a = a - B[base + j];
            else if (in_op == IN_A_PLUS_B) a = a + B[base + j];
            row[j + (j >> 5) * PADE] = a;
        }
        if (WEIGHTED) {
            const long long wbase = (f0 + fb) * (long long)(n - 1);
            T* wrow = wsm + (size_t)fb * npad;
            for (int j = tid; j < n; j += blockDim.x) wrow[j + (j >> 5) * PADE] = (j < n - 1) ? lamv[wbase + j] : T(0);
        }
    }
    if (use_tma) mbar_wait(&mbar, 0);
    __syncthreads();
    PHASE_MARK(0);

    // ---- scan: own chunk, then rounds until every lane has merged ----
    const int fb = tid / lpf, q = tid - fb * lpf;
    const bool lane_ok = fb < nfib && q < nchunks;
    const int fbc = lane_ok ? fb : 0;
    ChunkMasks m{mk + (size_t)fbc * lpf, mk + (size_t)(fpb + fbc) * lpf, mk + (size_t)(2 * fpb + fbc) * lpf};
    SmemLd32<T> y{smem_u32(ys + (size_t)fbc * npad)};
    T* xrow = X + (f0 + fbc) * (long long)n;
    GlobSt<T> stv{in_register(xrow)};
    RcpDiv<T> div{rcp};
    LaneState<T> st;
    st.active = false; st.finished = false; st.pend_a = -1; st.pend_k = K_NONE;

    const int nreg = in_register(n);
    auto phases = [&](auto lamf) {
        bool act = lane_ok ? walk_chunk<T, true, CHT>(q, 0, nchunks, nreg, y, stv, lamf, div, st, m) : false;
        int r = 1;
        for (; __syncthreads_or(act ? 1 : 0); r++) {
            if (r == 1) PHASE_MARK(1);
            act = lane_ok ? walk_chunk<T, false, CHT>(q, r, nchunks, nreg, y, stv, lamf, div, st, m) : false;
        }
        PHASE_MARK(2);
#ifdef PTV_PHASE_TIMING
        if (threadIdx.x == 0) { atomicAdd(&g_phase_ns[6], (unsigned long long)r); atomicAdd(&g_phase_ns[7], 1ull); }
#endif
    };
    if (WEIGHTED) phases(ArrayLam<T, SmemLd32<T>>{SmemLd32<T>{smem_u32(wsm + (size_t)fbc * npad)}});
    else if (LAMF) phases(UniformLam<T>{lamf[(f0 + fbc) / fpi]});
    else phases(UniformLam<T>{in_register(lam)});

    // ---- value of the segment entering each chunk (gathered before any output is written: the store is the output) ----
    const T cvq = lane_ok ? __ldcg(xrow + carry_of<CHT>(q, m)) : T(0);
    if (Mk) {
        // sparse result: the output row keeps only the segment values at their start positions; the chunk's start mask and the value
        // entering it go to Mk / Cv and the consumer (the fused tiled scatter, transpose.cu) expands the segments while it
        // transposes -- the fill phase (a fifth of this CTA's life) is not run at all
        if (CHT == 32) { if (lane_ok) { const long long e = (f0 + fbc) * (long long)lpf + q; Mk[e] = m.P[q]; Cv[e] = cvq; } }
        else if (lane_ok && !(q & 1)) {                             // per 32-sample window: the even chunk's lane writes both halves
            const long long e = (f0 + fbc) * (long long)nwin + (q >> 1);
            Mk[e] = m.P[q] | ((q + 1 < nchunks) ? (m.P[q + 1] << 16) : 0u); Cv[e] = cvq;
        }
        return;
    }
    if (lane_ok) cval[(size_t)fbc * lpf + q] = cvq;
    __syncthreads();
    PHASE_MARK(3);

    // ---- fill: 32-sample windows, FW per warp and batch: all sparse reads of the batch (segment values parked in the output
    //      row: L2 round trips that overlap), then its coalesced writes.  Reads of a window only touch that window, so batching
    //      windows is hazard free; the __syncwarp orders a window's reads before its own writes.  Larger batches
    //      overlap more round trips; FW >= 16 costs registers (a CTA less per SM). ----
    constexpr int FW = 8;
    const int warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
    const uint32_t below = 0xffffffffu >> (31 - lane);
    const int bpf = (nwin + FW - 1) / FW;                         // batches per fiber
    if (bpf >= nwarps) {                                          // long fibers: every warp has work inside each fiber
        for (int fb2 = 0; fb2 < nfib; fb2++) {
            const long long gb = (f0 + fb2) * (long long)n;
            const long long x2b = X2 ? ((f0 + fb2) / inc2) * inc2 * n + (f0 + fb2) % inc2 : 0;
            for (int c0 = warp * FW; c0 < nwin; c0 += nwarps * FW)
                fill_batch<T, FW, CL, CHT>(c0, nwin, nchunks, n, lane, below, X + gb, gb, x2b, mk + (size_t)fb2 * lpf, cval + (size_t)fb2 * lpf,
                                      ys + (size_t)fb2 * npad, out_op, A, B, C, X2, inc2);
        }
    } else {                                                      // short fibers: deal all (fiber, batch) pairs to the warps
        for (int bi = warp; bi < nfib * bpf; bi += nwarps) {
            const int fb2 = bi / bpf, c0 = (bi - fb2 * bpf) * FW;
            const long long gb = (f0 + fb2) * (long long)n;
            const long long x2b = X2 ? ((f0 + fb2) / inc2) * inc2 * n + (f0 + fb2) % inc2 : 0;
            fill_batch<T, FW, CL, CHT>(c0, nwin, nchunks, n, lane, below, X + gb, gb, x2b, mk + (size_t)fb2 * lpf, cval + (size_t)fb2 * lpf,
                                  ys + (size_t)fb2 * npad, out_op, A, B, C, X2, inc2);
        }
    }
    __syncthreads();
    PHASE_MARK(4);
    if (CL >= 1) {
        // ---- transposed second output, assembled from the G = fpb*CL adjacent fibers of this CTA / cluster: each group of G
        //      consecutive lanes writes G*sizeof(T) contiguous bytes (>= one full sector), positions split between the CTAs ----
        cg::cluster_group cluster = cg::this_cluster();
        __syncthreads();
        if (CL > 1) cluster.sync();
        const int rank = (CL > 1) ? (int)cluster.block_rank() : 0;
        const int G = fpb * CL;
        const long long fg0 = f0 - (long long)rank * fpb;                 // first fiber of the group
        const long long x2g = (fg0 / inc2) * inc2 * n + fg0 % inc2;
        const int jper = (n + CL - 1) / CL, jb = rank * jper, je = (jb + jper < n) ? jb + jper : n;
        for (int e = tid; e < (je - jb) * G; e += blockDim.x) {
            const int g2 = e % G, j = jb + e / G;
            const int owner = g2 / fpb, fbl = g2 - owner * fpb;
            const T* row = ys + (size_t)fbl * npad;
            if (CL > 1 && owner != rank) row = cluster.map_shared_rank(row, owner);
            X2[x2g + (long long)j * inc2 + g2] = row[j + (j >> 5) * PADE];
        }
        if (CL > 1) cluster.sync();                                       // nobody leaves while its rows may still be read
    }
}

// Returns cudaErrorInvalidConfiguration if the fibers do not fit in shared memory (caller falls back to the sequential kernel).
template <typename T>
static cudaError_t launch_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                         const T* lamv, cudaStream_t st, T* X2, long long inc2, uint32_t* Mk, T* Cv,
                                         const T* lamf = nullptr, long long fpi = 1) {
    if (g.inc != 1 || (lamf && (lamv || X2))) return cudaErrorInvalidConfiguration;
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    const int n = g.len;
    // 16-sample chunks for weighted float64 fibers: their second staged row (the weights) limits residency to 3 CTAs of 128
    // lanes per SM; twice the lanes per fiber bring the warps per SM back to 24
    const bool half = lamv && sizeof(T) == 8 && !X2 && (n + 15) / 16 <= 1024;
    const int nrows = (n + CH - 1) / CH;
    const int lpf = half ? (n + 15) / 16 : nrows;
    if (lpf > 1024) return cudaErrorInvalidConfiguration;
    const int npad = (n + (nrows + 1) * PadCfg<T>::PADE + PadCfg<T>::PADE - 1) / PadCfg<T>::PADE * PadCfg<T>::PADE;
    int fpb = (half ? 256 : 128) / lpf; if (fpb < 1) fpb = 1;
    if ((long long)fpb > g.nf) fpb = (int)g.nf;
    const bool cval_aliased = (size_t)fpb * lpf <= 2 * RCP_N;          // see the kernel
    const size_t per_fiber = (size_t)npad * sizeof(T) * (lamv ? 2 : 1) + (size_t)lpf * (12 + (cval_aliased ? 0 : sizeof(T)));
    const size_t smem = per_fiber * fpb + RCP_N * 2 * sizeof(T) + 16;
    if (smem > 200 * 1024) return cudaErrorInvalidConfiguration;
    int threads = ((fpb * lpf + 31) / 32) * 32;
    if (threads < RCP_N) threads = RCP_N;
    unsigned blocks = (unsigned)((g.nf + fpb - 1) / fpb);
    // TMA staging needs 16-byte aligned rows: aligned base, row pitch a multiple of 16 bytes, single input array
    const int use_tma = (op == IN_A) && (((uintptr_t)A & 15) == 0) && (((size_t)n * sizeof(T)) % 16 == 0);
    constexpr int SECT = 32 / (int)sizeof(T);                 // fibers per 32-byte sector
    using KernT = void (*)(const T*, const T*, const T*, int, T*, int, long long, int, T, const T*, int, int, int, int, T*, long long, uint32_t*, T*,
                           const T*, long long);
    KernT kern; int cl = 0;
    if (X2 && !lamv && threads <= 256 && inc2 > 0) {
        // sector-assembled transposed output: the CTA's own fibers suffice, or a cluster of SECT single-fiber CTAs
        if (fpb % SECT == 0 && g.nf % fpb == 0 && inc2 % fpb == 0) { kern = k_prox_chunked_contig<T, false, 256, 1>; cl = 1; }
        else if (fpb == 1 && g.nf % SECT == 0 && inc2 % SECT == 0) { kern = k_prox_chunked_contig<T, false, 256, SECT>; cl = SECT; }
        else kern = k_prox_chunked_contig<T, false, 256, 0>;
    } else {
        // small CTAs (<= 256 threads) get a register budget of up to 128/thread so loop constants stay in registers
        if (half) kern = threads <= 256 ? k_prox_chunked_contig<T, true, 256, 0, 16> : k_prox_chunked_contig<T, true, 1024, 0, 16>;
        else if (lamf) kern = threads <= 256 ? k_prox_chunked_contig<T, false, 256, 0, CH, true> : k_prox_chunked_contig<T, false, 1024, 0, CH, true>;
        else
        kern = threads <= 256 ? (lamv ? k_prox_chunked_contig<T, true, 256, 0> : k_prox_chunked_contig<T, false, 256, 0>)
                              : (lamv ? k_prox_chunked_contig<T, true, 1024, 0> : k_prox_chunked_contig<T, false, 1024, 0>);
    }
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    const long long inc2a = inc2 > 0 ? inc2 : 1;
    if (cl > 1) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        const int in_op_i = (int)op; const int use_tma_i = use_tma;
        uint32_t* mk0 = nullptr; T* cv0 = nullptr; const T* lf0 = nullptr; const long long fpi1 = 1;
        return cudaLaunchKernelEx(&cfg, kern, A, B, C, in_op_i, X, out_op, g.nf, n, lam, lamv, lpf, fpb, npad, use_tma_i, X2, inc2a, mk0, cv0, lf0, fpi1);
    }
    kern<<<blocks, threads, smem, st>>>(A, B, C, (int)op, X, out_op, g.nf, n, lam, lamv, lpf, fpb, npad, use_tma, X2, inc2a, Mk, Cv, lamf, fpi);
    return cudaGetLastError();
}

template <typename T>
cudaError_t prox_fibers_chunked_contig(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam,
                                       const T* lamv, cudaStream_t st, T* X2, long long inc2, const T* lamf, long long fpi) {
    return launch_chunked_contig<T>(A, B, C, op, X, out_op, g, lam, lamv, st, X2, inc2, nullptr, nullptr, lamf, fpi);
}
// Plain prox (OUT_X) of A (op) B with a SPARSE result: X only holds each segment's value at its start; Mk[fiber][chunk] = start mask,
// Cv[fiber][chunk] = value entering the chunk (chunks of 32 samples, (len + 31) / 32 per fiber).  See scatter_fibers_ex_sparse.
template <typename T>
cudaError_t prox_fibers_chunked_contig_sparse(const T* A, const T* B, InOp op, T* X, FiberGeom g, T lam, const T* lamv, uint32_t* Mk, T* Cv,
                                              cudaStream_t st, const T* lamf, long long fpi) {
    return launch_chunked_contig<T>(A, B, nullptr, op, X, OUT_X, g, lam, lamv, st, nullptr, 0, Mk, Cv, lamf, fpi);
}
template cudaError_t prox_fibers_chunked_contig_sparse<double>(const double*, const double*, InOp, double*, FiberGeom, double, const double*, uint32_t*,
                                                               double*, cudaStream_t, const double*, long long);
template cudaError_t prox_fibers_chunked_contig_sparse<float>(const float*, const float*, InOp, float*, FiberGeom, float, const float*, uint32_t*, float*,
                                                              cudaStream_t, const float*, long long);

template cudaError_t prox_fibers_chunked_contig<double>(const double*, const double*, const double*, InOp, double*, int, FiberGeom,
                                                        double, const double*, cudaStream_t, double*, long long, const double*, long long);
template cudaError_t prox_fibers_chunked_contig<float>(const float*, const float*, const float*, InOp, float*, int, FiberGeom,
                                                       float, const float*, cudaStream_t, float*, long long, const float*, long long);

// ------------------------------------------------------------------------------------------------------------------
// k_prox_chunked_strided: fibers with element stride `inc` whose neighbours are adjacent in memory (every dimension but
// the first of a column-major array).  A CTA takes FPB adjacent fibers: every global access then moves FPB*sizeof(T)
// contiguous bytes per sample position (32 B = one DRAM sector for FPB = 4 doubles / 8 floats), and the staging loop
// transposes on the fly into the same per-fiber padded rows the contiguous kernel uses, so the scan phases are shared.
// No transposed copy of the array is ever made.  The fill can fuse the second half of a Douglas-Rachford iteration
// (OUT_DR_ROWS*): it re-reads Y, s, t at the positions it writes; those lines were staged by this CTA moments ago and
// the working set of all resident CTAs (132 SMs x at most 3 CTAs x at most 72 KB of staged rows, < 30 MB) fits the 50 MB L2.
template <typename T> struct GlobStStrided {
    T* p; long long inc;
    __device__ __forceinline__ void operator()(int j, T v) const { p[(long long)j * inc] = v; }
};

template <typename T, int FPB>
__global__ void __launch_bounds__(1024) k_prox_chunked_strided(const T* __restrict__ A, const T* __restrict__ B, const T* __restrict__ C,
                                                           int in_op, T* __restrict__ X, int out_op, long long nf, int n, long long inc,
                                                           T lam, int lpf, int npad, T* __restrict__ V) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    RcpPair<T>* rcp = reinterpret_cast<RcpPair<T>*>(smem_raw);
    T* ys = reinterpret_cast<T*>(rcp + RCP_N);                    // [FPB][npad]
    T* cval = ys + (size_t)FPB * npad;                            // [FPB][lpf]
    uint32_t* mk = reinterpret_cast<uint32_t*>(cval + (size_t)FPB * lpf);      // [3][FPB][lpf]
    constexpr int PADE = PadCfg<T>::PADE;
    constexpr int CPW = 32 / FPB;                                 // sample positions one warp covers per access
    const int tid = threadIdx.x;
    const long long f0 = (long long)blockIdx.x * FPB;             // first fiber of the group (inc % FPB == 0: one slab)
    const long long base0 = (f0 / inc) * inc * n + (f0 % inc);
    const int nchunks = (n + CH - 1) / CH;

    // ---- stage: thread (r, cc) reads fiber r at positions cc, cc + step, ...; FPB lanes share one sector ----
    if (tid < RCP_N) { rcp[tid].r = tid ? T(1) / T(tid) : T(0); rcp[tid].d = T(tid); }
    {
        const int r = tid % FPB, cc = tid / FPB, step = blockDim.x / FPB;
        T* row = ys + (size_t)r * npad;
        constexpr int U = 8;                                      // loads in flight per thread and array
        for (int k0 = cc; k0 < n; k0 += step * U) {
            T a[U], b[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int k = k0 + u * step;
                const long long g = base0 + (long long)k * inc + r;
                a[u] = (k < n) ? A[g] : T(0);
                b[u] = (k < n && in_op != IN_A) ? B[g] : T(0);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int k = k0 + u * step;
                T v = a[u];
                if (in_op == IN_A_MINUS_B) v = v - b[u]; else if (in_op == IN_A_PLUS_B) v = v + b[u];
                if (k < n) row[k + (k >> 5) * PADE] = v;
            }
        }
    }
    __syncthreads();

    // ---- scan (shared with the contiguous kernel) ----
    const int fb = tid / lpf, q = tid - fb * lpf;
    const bool lane_ok = fb < FPB && q < nchunks;
    const int fbc = lane_ok ? fb : 0;
    ChunkMasks m{mk + (size_t)fbc * lpf, mk + (size_t)(FPB + fbc) * lpf, mk + (size_t)(2 * FPB + fbc) * lpf};
    SmemLd32<T> y{smem_u32(ys + (size_t)fbc * npad)};
    // sparse value store: a contiguous scratch row per fiber (V, [fiber][n]) when the caller provides one -- the values are
    // written and read back by this CTA only, so a dense row keeps them in a handful of L2 lines -- else the output itself
    T* xfib = V ? V + (f0 + fbc) * (long long)n : X + base0 + fbc;
    const long long vinc = V ? 1 : inc;
    GlobStStrided<T> stv{xfib, vinc};
    RcpDiv<T> div{rcp};
    LaneState<T> st;
    st.active = false; st.finished = false; st.pend_a = -1; st.pend_k = K_NONE;
    UniformLam<T> lamf{in_register(lam)};
    const int nreg = in_register(n);
    {
        bool act = lane_ok ? walk_chunk<T, true>(q, 0, nchunks, nreg, y, stv, lamf, div, st, m) : false;
        for (int r = 1; __syncthreads_or(act ? 1 : 0); r++)
            act = lane_ok ? walk_chunk<T, false>(q, r, nchunks, nreg, y, stv, lamf, div, st, m) : false;
    }
    if (lane_ok) cval[(size_t)fbc * lpf + q] = __ldcg(xfib + (long long)carry_of(q, m) * vinc);
    __syncthreads();

    // ---- fill: a warp takes one 32-sample window of all FPB fibers: FPB accesses of CPW positions x FPB fibers each; all
    //      sparse reads of the window first, then its writes (FPB*sizeof(T)-byte pieces, sector aligned) ----
    const int warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
    const int r = lane % FPB, jj = lane / FPB;
    const uint32_t* Pm = mk + (size_t)r * lpf;
    const T* cv = cval + (size_t)r * lpf;
    const T* yr = ys + (size_t)r * npad;
    const T* vr = V ? V + (f0 + r) * (long long)n : X + base0 + r;
    for (int c = warp; c < nchunks; c += nwarps) {
        T v[FPB];
        const uint32_t pw = Pm[c];
#pragma unroll
        for (int u = 0; u < FPB; u++) {
            const int b = u * CPW + jj, k = (c << 5) + b;
            v[u] = T(0);
            if (k < n) {
                const uint32_t w = pw & (0xffffffffu >> (31 - b));
                v[u] = w ? __ldcg(vr + (long long)((c << 5) + high_bit(w)) * vinc) : cv[c];
            }
        }
        __syncwarp();
#pragma unroll
        for (int u = 0; u < FPB; u++) {
            const int b = u * CPW + jj, k = (c << 5) + b;
            if (k < n) {
                const long long g = base0 + (long long)k * inc + r;
                X[g] = apply_out_ex<T>(out_op, yr[k + c * PADE], v[u], A, B, C, g);
            }
        }
    }
}

template <typename T, int FPB>
static cudaError_t launch_strided(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, T* V, cudaStream_t st) {
    const int n = g.len;
    const int lpf = (n + CH - 1) / CH;
    const int npad = (n + (lpf + 1) * PadCfg<T>::PADE + PadCfg<T>::PADE - 1) / PadCfg<T>::PADE * PadCfg<T>::PADE;
    const size_t smem = (size_t)FPB * ((size_t)npad * sizeof(T) + (size_t)lpf * (12 + sizeof(T))) + RCP_N * 2 * sizeof(T) + 16;
    const int threads = ((FPB * lpf + 31) / 32) * 32;
    if (smem > 220 * 1024 || threads > 1024 || g.inc % FPB != 0 || g.nf % FPB != 0) return cudaErrorInvalidConfiguration;
    auto kern = k_prox_chunked_strided<T, FPB>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    kern<<<(unsigned)(g.nf / FPB), threads < RCP_N ? RCP_N : threads, smem, st>>>(A, B, C, (int)op, X, out_op, g.nf, n, g.inc, lam, lpf, npad, V);
    return cudaGetLastError();
}

// Returns cudaErrorInvalidConfiguration when the shape does not suit this kernel (caller falls back).
template <typename T>
cudaError_t prox_fibers_chunked_strided(const T* A, const T* B, const T* C, InOp op, T* X, int out_op, FiberGeom g, T lam, T* V,
                                        cudaStream_t st) {
    if (g.inc <= 1) return cudaErrorInvalidConfiguration;
    if (g.nf <= 0 || g.len <= 0) return cudaSuccess;
    constexpr int SECT = 32 / (int)sizeof(T);        // fibers per 32-byte sector: 4 doubles, 8 floats
    // Group width: as wide as possible while at least three CTAs stay resident per SM (the kernel is latency/issue bound,
    // not bandwidth bound, so occupancy beats access width); half a sector per access is the floor -- the neighbouring CTA
    // takes the other half at the same time and finds it in L2.
    const int lpf = (g.len + CH - 1) / CH;
    const size_t per_fiber = (size_t)(g.len + (lpf + 2) * PadCfg<T>::PADE) * sizeof(T) + (size_t)lpf * (12 + sizeof(T));
    const size_t budget = 72 * 1024;
    cudaError_t e = cudaErrorInvalidConfiguration;
    if (per_fiber * 4 * SECT <= budget) e = launch_strided<T, 4 * SECT>(A, B, C, op, X, out_op, g, lam, V, st);
    if (e == cudaErrorInvalidConfiguration && per_fiber * 2 * SECT <= budget) { cudaGetLastError(); e = launch_strided<T, 2 * SECT>(A, B, C, op, X, out_op, g, lam, V, st); }
    if (e == cudaErrorInvalidConfiguration && per_fiber * SECT <= budget) { cudaGetLastError(); e = launch_strided<T, SECT>(A, B, C, op, X, out_op, g, lam, V, st); }
    if (e == cudaErrorInvalidConfiguration) { cudaGetLastError(); e = launch_strided<T, SECT / 2>(A, B, C, op, X, out_op, g, lam, V, st); }
    if (e == cudaErrorInvalidConfiguration) { cudaGetLastError(); e = launch_strided<T, SECT>(A, B, C, op, X, out_op, g, lam, V, st); }
    return e;
}
template cudaError_t prox_fibers_chunked_strided<double>(const double*, const double*, const double*, InOp, double*, int, FiberGeom, double, double*, cudaStream_t);
template cudaError_t prox_fibers_chunked_strided<float>(const float*, const float*, const float*, InOp, float*, int, FiberGeom, float, float*, cudaStream_t);

}  // namespace ptv

#ifdef PTV_PHASE_TIMING
extern "C" void proxtv_debug_phase_read(unsigned long long* out, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, ptv::g_phase_ns, sizeof(unsigned long long) * 8);
    if (reset) { unsigned long long z[8] = {0}; cudaMemcpyToSymbol(ptv::g_phase_ns, z, sizeof(z)); }
}
#endif
