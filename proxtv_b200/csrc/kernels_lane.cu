// kernels_lane.cu -- the lane-per-fiber streaming TV-L1 prox kernel for sm_90a (H100) (algorithm and shared code: lane_core.cuh).
//
// One warp = 32 adjacent fibers x one chunk of rows.  Rows enter the warp's circular shared-memory window as TMA tiles
// (cp.async.bulk.tensor, one mbarrier per tile slot; SASS: UTMALDG), the 32 lanes scan their own window column (bank-conflict
// free), and finished rows leave through the drain:
//     STRIDED layout (fibers adjacent in memory: every dimension but the first of a column-major array)
//         a window row IS one contiguous 32-sample line of the array: the tile lands in place, rows are drained with one
//         coalesced store each -- no transposed copy of anything (this replaces the gather / scatter kernels of transpose.cu)
//     CONTIG layout (fibers contiguous: the first dimension)
//         a TMA box of 16 rows x 32 fibers lands fiber-major with the 128-byte hardware swizzle and is transposed into the window
//         by the warp; finished boxes are transposed back and leave with a TMA store (UTMASTG)
// Fused Douglas-Rachford arithmetic (PassOp) sits either at the landing (staged ops: three operand tiles combined into the scan's
// input) or in the drain (operands fetched with coalesced loads one epoch ahead); drain-side ops can write their results TRANSPOSED
// -- fiber-major -- through an in-place exchange of the 32 x 8 block just swept (store8_transposed), which is what lets both passes of
// a 2D iteration be STRIDED passes over two copies in opposite layouts (solver.cu: dr2_lane_t_body).
// No CTA-wide barrier after the prologue: warps are independent (a CTA is NW of them sharing the reciprocal table; NW = 4, one per SM
// sub-partition, three CTAs per SM when the pass needs no staging).
#include "ptv_internal.h"
#include "lane_core.cuh"
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

namespace ptvl {

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// non-blocking poll (try_wait may suspend the thread for a while before it reports failure; test_wait never does)
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(s32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
// same with an L2 cache policy (createpolicy) for the lines the load brings in
__device__ __forceinline__ void tma_load_3d_hint(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;"
                 ::"r"(s32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(s32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(map), "r"(s32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- kernel arguments
// Fused pass arithmetic.  Two generations of the Douglas-Rachford forms:
//   LOP_DR_B / LOP_DR_B_FINAL  "staged": the row pass combines three operand tiles when they land (in = Y - (2 (t - x1) - t)); costs
//                              8 KB of staging per warp, i.e. a third of the resident warps
//   LOP_DRA / _FINAL / LOP_DRB "transposed": every pass lands plain tiles, does its arithmetic in the DRAIN (operands read with
//                              coalesced loads, one epoch ahead) and writes its results TRANSPOSED, so that both passes of an
//                              iteration are strided passes -- one over the row-major copies, one over the column-major ones
enum LaneOp { LOP_PLAIN = 0, LOP_DR_B = 1, LOP_DR_B_FINAL = 2, LOP_DRA = 3, LOP_DRA_FINAL = 4, LOP_DRB = 5, LOP_PLAIN_T = 6 /* plain, result transposed */ };
template <int OP> struct OpTraits {
    static constexpr bool staged = OP == LOP_DR_B || OP == LOP_DR_B_FINAL;           // B, C tiles combined at landing
    static constexpr bool tout = OP >= LOP_DRA;                                     // results written transposed (fiber-major)
    static constexpr bool two_out = OP == LOP_DRA;                                  // second result array X2
    static constexpr int drain_reads = (OP == LOP_DR_B || OP == LOP_DRA || OP == LOP_DRA_FINAL) ? 2 : (OP == LOP_DRB ? 1 : 0);
};

template <typename T> struct LaneArgs {
    CUtensorMap tmA, tmB, tmC;      // loads (B, C only for the fused Douglas-Rachford forms)
    CUtensorMap tmX;                // store (CONTIG layout)
    const T* A; const T* B; const T* C; T* X; T* X2;
    long long inc;                  // fiber stride (STRIDED: fibers per slab; CONTIG: 1)
    long long per_slab;             // fibers per slab (STRIDED: inc; CONTIG: nf)
    int slabs, gps;                 // groups of 32 fibers per slab
    TaskPlan plan;
    T lam;
    acc_t lamc[2];                  // 2 lam, -2 lam (float64: what the scan adds / resets to)
    int* rec;                       // [5][plan.nmax][slabs*gps*32] chunk records (in, out, overflow, in2, in3)
    int* group_count;               // [slabs*gps] finished-task counters (self-resetting)
    unsigned long long* stats;      // [0] repair scans, [1] retired lanes
    unsigned long long* tlog;       // optional (tools): per task TLOG_WORDS words, see k_lane
    long long ntasks;
    const T* lamf; long long fpi;   // per-fiber penalties (the LAMF instantiations): fiber j's is lamf[j / fpi], in place of lam
};
constexpr int TLOG_WORDS = 16;

// fused arithmetic of a pass: what a lane scans (in) and what it writes for prox value x (out)
template <typename T, int OP> struct PassOp {
    // what a lane scans, from the landed tiles (staged forms only; every other form scans A as it is)
    static __device__ __forceinline__ T in(T a, T b, T c) {
        if (!OpTraits<OP>::staged) return a;
        return in_d(a, c - b, c);                            // d = t - prox_cols(t)          (src/TV2Dopt.cpp:545-546)
    }
    // the same from d = c - b, rounded once (the landing keeps it for the drain: out_d)
    static __device__ __forceinline__ T in_d(T a, T d, T c) {
        if (OP == LOP_DR_B) return a - (T(2) * d - c);       // Y - s, s = 2 (t - x) - t      (:411, :515)
        return a - d;                                        // final: s = t - x              (:427)
    }
    // what the drain writes for prox value x and the operands b, c read at the drained position: o1 -> X, o2 -> X2
    static __device__ __forceinline__ void out(T x, T b, T c, T& o1, T& o2) {
        o2 = T(0);
        if (OP == LOP_DR_B) o1 = (c - b) + x;                // t' = 0.5 (t + s + 2 prox_rows(Y - s)) = (t - x_cols) + x_rows   (:419-422)
        else if (OP == LOP_DRA) { const T d = c - x; o2 = d; o1 = b - (T(2) * d - c); }   // b = Y, c = t: d = t - x_cols, u = Y - (2 d - t)
        else if (OP == LOP_DRA_FINAL) o1 = b - (c - x);      // u = Y - (t - x_cols)          (:427)
        else if (OP == LOP_DRB) o1 = b + x;                  // b = d: t' = (t - x_cols) + x_rows
        else o1 = x;
    }
    // LOP_DR_B from the d the landing computed: (c - b) + x above, on the same rounded c - b
    static __device__ __forceinline__ T out_d(T x, T d) { return d + x; }
};

// d = t - x1 of the staged row pass (LOP_DR_B), carried in registers from the landing of a tile to its drain instead of being read
// again from global memory.  One slot of 8 values per lane and tile slot of the window (W / 8 slots), indexed by the ABSOLUTE tile
// index row0 / 8 -- the window's ring position: halo tiles and tiles past the chunk's end are landed but never drained, so
// push / pop counters would drift -- and the window itself keeps a slot from being landed again before its rows are swept (a tile
// is requested only when row_req + 8 <= row_lo + W, and row_lo <= the next row to sweep).  The slot is warp-uniform; every access
// goes through at(), whose cases name the slot's registers at compile time, so that the ring stays in registers.  512 bytes per
// lane (128 registers) for float64 with a 64-row window and float32 with a 128-row one; larger rings keep the re-reading drain.
template <typename T, int W, int OP> struct DRing {
    static constexpr int NS = W / 8;
    static constexpr bool on = OP == LOP_DR_B && NS * 8 * (int)sizeof(T) <= 512;
    T d[on ? NS : 1][8];
    __device__ __forceinline__ static unsigned slot(int row0) { return ((unsigned)row0 / 8u) % (unsigned)NS; }
    // f(d[k]) for the slot k of the tile at row0: one case per slot, each with its own copy of f working on its own registers, so
    // that selecting the slot is a jump (the whole landing combine or drain store of a tile is inside f: a body too large to be
    // turned into selects over every slot, which a bare copy in and out of the ring would be)
    template <class F> __device__ __forceinline__ void at(int row0, F f) {
        if constexpr (on) {
#define PTV_RING_CASE(k) case k: if constexpr (k < NS) f(d[k < NS ? k : 0]); break;
            switch (slot(row0)) {
                PTV_RING_CASE(0) PTV_RING_CASE(1) PTV_RING_CASE(2) PTV_RING_CASE(3) PTV_RING_CASE(4) PTV_RING_CASE(5) PTV_RING_CASE(6)
                PTV_RING_CASE(7) PTV_RING_CASE(8) PTV_RING_CASE(9) PTV_RING_CASE(10) PTV_RING_CASE(11) PTV_RING_CASE(12) PTV_RING_CASE(13)
                PTV_RING_CASE(14) PTV_RING_CASE(15)
                default: break;
            }
#undef PTV_RING_CASE
        }
    }
};

// ---------------------------------------------------------------- the scan loop, device form
// Same arithmetic and the same decisions as Lane<T>::run (lane_core.cuh, the form the CPU emulation executes), with positions
// carried pre-multiplied by the window row pitch so that a window access is ONE logic op + the shared-memory instruction:
//     address(row) = (((row * ROWB) & (W * ROWB - 1)) | lane offset) + window base
template <typename T> struct SmemIO { };
template <> struct SmemIO<double> {
    static __device__ __forceinline__ double ld(uint32_t a) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a)); return v; }
    static __device__ __forceinline__ void st(uint32_t a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
};
template <> struct SmemIO<float> {
    static __device__ __forceinline__ float ld(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a)); return v; }
    static __device__ __forceinline__ void st(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
};
__device__ __forceinline__ void opaque(double& v) { asm volatile("" : "+d"(v)); }
__device__ __forceinline__ void opaque(float& v) { asm volatile("" : "+f"(v)); }
__device__ __forceinline__ void sts_u8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts_u8_pred(uint32_t a, int v, bool p) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.shared.u8 [%0], %1;\n\t}" ::"r"(a), "r"(v), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ void sts_val_pred(uint32_t a, double v, bool p) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.shared.f64 [%0], %1;\n\t}" ::"r"(a), "d"(v), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ void sts_val_pred(uint32_t a, float v, bool p) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.shared.f32 [%0], %1;\n\t}" ::"r"(a), "f"(v), "r"((uint32_t)p) : "memory");
}
// value + flag byte, both under one predicate (kept as predicated stores: the compiler would otherwise branch around them)
__device__ __forceinline__ void sts_pred(uint32_t va, double v, uint32_t fa, bool p) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %3, 0;\n\t@q st.shared.f64 [%0], %1;\n\t@q st.shared.u8 [%2], 1;\n\t}"
                 ::"r"(va), "d"(v), "r"(fa), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ void sts_pred(uint32_t va, float v, uint32_t fa, bool p) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %3, 0;\n\t@q st.shared.f32 [%0], %1;\n\t@q st.shared.u8 [%2], 1;\n\t}"
                 ::"r"(va), "f"(v), "r"(fa), "r"((uint32_t)p) : "memory");
}

template <typename T, int W> struct DevWin {
    static constexpr int ROWB = LANES * (int)sizeof(T);          // bytes per window row
    static constexpr uint32_t MASK = (uint32_t)(W * ROWB - 1) & ~(uint32_t)(ROWB - 1);
    static constexpr int SH = (ROWB == 256) ? 5 : 4;             // (k * ROWB) >> SH == k * 8: byte offset into the float64 reciprocal table
    static constexpr int FSH = (ROWB == 256) ? 8 : 7;            // scaled position -> row (positions are exact multiples: arithmetic shift)
    uint32_t wbase;    // shared address of the warp's window (a kernel constant when the CTA is a single warp: folds into the access)
    uint32_t lane8;    // byte offset of this lane's column inside a window row
    uint32_t flg;      // shared address of this lane's flag bytes
    uint32_t rcp;      // shared address of the reciprocal table
    __device__ __forceinline__ uint32_t flag_at(int pos) const { return flg + (((uint32_t)pos >> FSH) & (uint32_t)(W - 1)); }
    __device__ __forceinline__ uint32_t at(int pos) const {
        uint32_t o;                                    // (pos & MASK) | lane8 in one LOP3 (the two fields never overlap)
        asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(o) : "r"((uint32_t)pos), "r"(MASK), "r"(lane8));
        return o + wbase;
    }
};

template <bool PH1, typename T, int W>
__device__ __forceinline__ void run_dev(Lane<T>& L, const DevWin<T, W> dw, const TaskGeom& g, const acc_t lam2, const acc_t nlam2, int niter) {
    using DW = DevWin<T, W>;
    constexpr int ROWB = DW::ROWB;
    acc_t Z = L.Z, lo = L.lo, hi = L.hi;
    int ia = L.i << DW::FSH, la = L.last << DW::FSH, bloa = L.blo << DW::FSH, bhia = L.bhi << DW::FSH, in_ = L.in_rec;
    const int csa = g.cs << DW::FSH;
    // unrolled by two: the loop-carried registers swap roles instead of being copied; 2 lam / -2 lam come from the constant bank
#pragma unroll 2
    for (int it = 0; it < niter; it++) {
        const acc_t y = (acc_t)SmemIO<T>::ld(dw.at(ia));
        const int ka = ia - la;
        const acc_t r = SmemIO<double>::ld(dw.rcp + ((uint32_t)ka >> DW::SH));
        // both slopes straight from the old sum (ch does not wait for cl: the float64 dependency chain is add -> multiply -> compare)
        const acc_t cl = (Z + y) * r, ch = (Z + (y + lam2)) * r;
        Z += y;
        const bool first = (ka == ROWB);
        const bool can = !first;
        const bool craw = lo > ch, fraw = hi < cl;          // both compares issue back to back (neither waits for the other)
        const bool cbk = can & craw;
        const bool fbk = can & !craw & fraw;
        const bool brk = cbk | fbk;
        const int ea = cbk ? bloa : bhia;
        const int fa = la + ROWB;
        // the finished segment's value goes to its first (owned) row; the new segment gets its start mark (kind + 1)
        bool em = brk; int fea = fa;
        if (PH1) {
            em = brk & (ea >= csa);
            fea = fa > csa ? fa : csa;
            const uint32_t kf = lds_u8(dw.flag_at(fa));
            in_ = (em & (in_ == REC_NONE)) ? rec_pack(fa >> DW::FSH, (int)kf - 1) : in_;
            sts_u8_pred(dw.flag_at(fea), LK_BEGIN + 1, em & (fea != fa));      // clipped: the sweep needs a start mark at cs
        }
        const uint32_t va = dw.at(fea);
        sts_val_pred(va, (T)lo, em & cbk);
        sts_val_pred(va, (T)hi, em & fbk);
        const uint32_t nfl = dw.flag_at(ea + ROWB);
        sts_u8_pred(nfl, LK_CEIL + 1, cbk);
        sts_u8_pred(nfl, LK_FLOOR + 1, fbk);
        const bool tlo = first | (cl >= lo), thi = first | (ch <= hi);
        lo = tlo ? cl : lo; bloa = tlo ? ia : bloa;
        hi = thi ? ch : hi; bhia = thi ? ia : bhia;
        Z = cbk ? 0.0 : (fbk ? nlam2 : Z);
        ia = (brk ? ea : ia) + ROWB;
        la = brk ? ea : la;
    }
    L.Z = Z; L.lo = lo; L.hi = hi; L.i = ia >> DW::FSH; L.last = la >> DW::FSH; L.blo = bloa >> DW::FSH; L.bhi = bhia >> DW::FSH;
    L.in_rec = in_;
}

// LAMF: the lane's own penalty; scan() then takes 2 lam, -2 lam from the lam2 it is given (the same values lamc would hold for it)
template <typename T, int W, bool LAMF = false> struct DevEnv {
    Lane<T> L; int lane; DevWin<T, W> dw; const acc_t* lamc;      // lamc: {2 lam, -2 lam} in the kernel's parameter block (constant bank)
    template <class F> __device__ __forceinline__ void each(F f) { f(L, lane); }
    template <class F> __device__ __forceinline__ int rmin(F f) { return __reduce_min_sync(0xffffffffu, f(L, lane)); }
    template <class F> __device__ __forceinline__ int rmax(F f) { return __reduce_max_sync(0xffffffffu, f(L, lane)); }
    template <class F> __device__ __forceinline__ bool any(F f) { return __any_sync(0xffffffffu, f(L, lane)); }
    __device__ __forceinline__ void sync() { __syncwarp(); }
    __device__ __forceinline__ void scan(Lane<T>& l, const Window<T, W>&, int, const TaskGeom& g, const acc_t*, acc_t lam2, bool ph1, int niter) {
        if constexpr (LAMF) { if (ph1) run_dev<true, T, W>(l, dw, g, lam2, -lam2, niter); else run_dev<false, T, W>(l, dw, g, lam2, -lam2, niter); }
        else { if (ph1) run_dev<true, T, W>(l, dw, g, lamc[0], lamc[1], niter); else run_dev<false, T, W>(l, dw, g, lamc[0], lamc[1], niter); }
    }
};
// a lane's own penalty, as warp_task takes it per lane (each thread of the warp is one lane)
template <typename T> struct LaneLam { T v; __device__ __forceinline__ T operator()(int) const { return v; } };
// the penalty of fiber j of a LAMF launch
template <typename T> __device__ __forceinline__ T fiber_lam(const LaneArgs<T>& a, long long j) { return a.lamf[j / a.fpi]; }

// ---------------------------------------------------------------- STRIDED layout: feed and drain
template <typename T, int W, int RT, int OP> struct FeedStrided {
    static constexpr int R = RT;
    static constexpr int NST = 2;                       // staging tiles for the B / C operands of the fused forms
    static constexpr int MAXQ = OpTraits<OP>::staged ? NST : W / RT;
    static constexpr int NBAR = W / RT;
    using Ring = DRing<T, W, OP>;
    static_assert(!Ring::on || RT == 8, "the d ring holds one 8-row drain group per tile");
    const LaneArgs<T>* a; T* win; T* stB; T* stC; uint64_t* bar; int x0, z, q0, lane;
    Ring* ring;                                         // d = t - x1 of the landed tiles (Ring::on), read by the drain
    template <class Env> __device__ __forceinline__ void request(Env&, int row0) {
        __syncwarp();
        if (lane == 0) {
            fence_proxy_async();                        // the slot's last generic-proxy accesses precede the async write
            const int q = (int)((unsigned)row0 / (unsigned)R) - q0;
            uint64_t* b = bar + ((unsigned)q % (unsigned)NBAR);
            mbar_expect_tx(b, (uint32_t)(R * LANES * sizeof(T) * (OpTraits<OP>::staged ? 3 : 1)));
            // the scan's input is read again by the drain only in the LOP_DRA forms (C == A); everywhere else its lines are dead once
            // they have landed: evict-first, so that what L2 keeps are the operand tiles the drain will come back for
            if (OP == LOP_DRA || OP == LOP_DRA_FINAL) tma_load_3d(win + ((row0 & (W - 1)) << 5), &a->tmA, x0, row0, z, b);
            else tma_load_3d_hint(win + ((row0 & (W - 1)) << 5), &a->tmA, x0, row0, z, b, policy_evict_first());
            if (OpTraits<OP>::staged) {
                // with the d ring the drain does not come back for B and C either (LOP_DR_B_FINAL never does): single use
                if (Ring::on || OP == LOP_DR_B_FINAL) {
                    tma_load_3d_hint(stB + (q % NST) * R * LANES, &a->tmB, x0, row0, z, b, policy_evict_first());
                    tma_load_3d_hint(stC + (q % NST) * R * LANES, &a->tmC, x0, row0, z, b, policy_evict_first());
                } else {
                    tma_load_3d(stB + (q % NST) * R * LANES, &a->tmB, x0, row0, z, b);
                    tma_load_3d(stC + (q % NST) * R * LANES, &a->tmC, x0, row0, z, b);
                }
            }
        }
    }
    template <class Env> __device__ __forceinline__ bool landed(Env&, int row0, bool block) {
        const unsigned q = (unsigned)row0 / (unsigned)R - (unsigned)q0;
        uint64_t* b = bar + (q % (unsigned)NBAR);
        const uint32_t parity = (uint32_t)((q / (unsigned)NBAR) & 1u);
        // the decision must be warp-uniform (it steers the task's control flow), and every lane needs the acquire of its own
        // successful wait before it reads the tile: all lanes poll, the vote decides
        bool ok = __all_sync(0xffffffffu, mbar_test(b, parity));
        if (!ok && !block) return false;
        while (!ok) ok = __all_sync(0xffffffffu, mbar_try(b, parity));
        if (OpTraits<OP>::staged) {
            const T* sb = stB + (q % NST) * R * LANES; const T* sc = stC + (q % NST) * R * LANES;
            T* wr = win + ((row0 & (W - 1)) << 5);
            auto combine = [&](T* d) {
#pragma unroll
                for (int r = 0; r < R; r++) {
                    const T c = sc[r * LANES + lane];
                    d[r] = c - sb[r * LANES + lane];
                    wr[r * LANES + lane] = PassOp<T, OP>::in_d(wr[r * LANES + lane], d[r], c);
                }
            };
            if constexpr (Ring::on) ring->at(row0, combine);          // d of this tile kept in its ring slot
            else { T d[R]; combine(d); }
        }
        __syncwarp();
        return true;
    }
};

template <typename T> struct Vec16 { };
template <> struct Vec16<double> {
    static __device__ __forceinline__ void ld(uint32_t a, double* v) { asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v[0]), "=d"(v[1]) : "r"(a)); }
    static __device__ __forceinline__ void st(uint32_t a, const double* v) { asm volatile("st.shared.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(v[0]), "d"(v[1]) : "memory"); }
};
template <> struct Vec16<float> {
    static __device__ __forceinline__ void ld(uint32_t a, float* v) { asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "r"(a)); }
    static __device__ __forceinline__ void st(uint32_t a, const float* v) { asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory"); }
};


// L2 eviction priorities of the drain: everything the drain touches is a LAST use inside this kernel -- results are written once and
// not read again here, operands are read once (or re-read: the scan's own input, landed by TMA a window earlier) -- so its loads and
// stores are marked evict-first; what stays in L2 are the tiles that were landed but not yet drained, i.e. exactly the re-reads.
__device__ __forceinline__ void st_global_v16(double* p, const double* v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v[0]), "d"(v[1]), "l"(pol) : "memory"); }
__device__ __forceinline__ void st_global_v16(float* p, const float* v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "l"(pol) : "memory"); }
__device__ __forceinline__ void st_stream(double* p, double v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory"); }
__device__ __forceinline__ void st_stream(float* p, float v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory"); }
__device__ __forceinline__ double ld_last(const double* p, uint64_t pol) { double v; asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol)); return v; }
__device__ __forceinline__ float ld_last(const float* p, uint64_t pol) { float v; asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol)); return v; }

// 8 results per lane (rows r0 .. r0+7 of 32 adjacent fibers) written TRANSPOSED -- dst[f * n + r], fiber-major -- without any extra
// shared memory: the window rows just swept are dead, so their 32 x 8 block is rewritten fiber-major in place (16-byte chunks,
// chunk c of fiber f at position c ^ s(f): conflict-free on both sides) and read back so that NCH adjacent lanes hold the 8
// consecutive results of ONE fiber; a store instruction then covers 32 / NCH fibers x one full 64-byte (f64) / 32-byte (f32) run instead
// of 32 scattered 16-byte pieces.  dst points at (fiber 0 of the group, row r0); fibers >= nvalid are not written.
template <typename T, int W>
__device__ __forceinline__ void store8_transposed(const Window<T, W>& w, int r0, int lane, const T* xs, T* dst, long long n, int nvalid, uint64_t pol) {
    constexpr int EPC = 16 / (int)sizeof(T), NCH = 8 / EPC, FB = 8 * (int)sizeof(T), FPI = LANES / NCH, SG = 8 / NCH;
    const uint32_t reg = s32(w.win) + (uint32_t)(((r0 & (W - 1)) << 5) * (int)sizeof(T));
    __syncwarp();                                        // every lane has read its column of these rows
#pragma unroll
    for (int c = 0; c < NCH; c++) Vec16<T>::st(reg + (uint32_t)(lane * FB + ((c ^ ((lane / SG) & (NCH - 1))) << 4)), xs + c * EPC);
    __syncwarp();
    const int cc = lane % NCH;
#pragma unroll
    for (int k = 0; k < NCH; k++) {
        const int f = lane / NCH + FPI * k;
        T v[EPC];
        Vec16<T>::ld(reg + (uint32_t)(f * FB + ((cc ^ ((f / SG) & (NCH - 1))) << 4)), v);
        if (f < nvalid) st_global_v16(dst + (long long)f * n + cc * EPC, v, pol);
    }
    __syncwarp();                                        // the block may be rewritten (second output, next tile)
}

template <typename T, int W, int OP> struct DrainStrided {
    using TR = OpTraits<OP>;
    using Ring = DRing<T, W, OP>;
    // operand loads of a whole group: none when the feed's d ring holds what they would bring (the partial last group and the
    // repair path still read B and C)
    static constexpr int group_reads = Ring::on ? 0 : TR::drain_reads;
    const T* __restrict__ B; const T* __restrict__ C; T* __restrict__ X; T* __restrict__ X2;
    Ring* ring;
    long long gbase, stride;          // this lane's fiber: element of row 0, element stride between rows
    int ce;                           // end of the chunk (rows beyond are not this task's)
    long long tbase, n; int nvalid;   // transposed results: element (fiber 0 of the group, row 0) of the fiber-major array; fibers in the group
    // operands of the fused drain arithmetic for the group of rows that will be swept next, fetched one epoch ahead (coalesced: a
    // window row is one contiguous line of every operand array)
    T pb[8], pc[8]; int pf_row; uint64_t pol;     // pol: L2 evict-first policy of the drain's loads and stores
    __device__ __forceinline__ void fetch(int r0) {
        const long long g0 = gbase + (long long)r0 * stride;
        const T* __restrict__ qb = B + g0; const T* __restrict__ qc = C + g0;
#pragma unroll
        for (int u = 0; u < 8; u++) { pb[u] = ld_last(qb, pol); qb += stride; if (TR::drain_reads > 1) { pc[u] = ld_last(qc, pol); qc += stride; } }
    }
    __device__ __forceinline__ void prefetch(int r0, int ce, bool valid) {
        if (group_reads == 0 || !valid || r0 + 8 > ce || r0 == pf_row) return;
        fetch(r0); pf_row = r0;
    }
    __device__ __forceinline__ void rows8(const Window<T, W>& w, int r0, int cnt, int lane, const T* xs, bool valid) {
        if (!valid && !(TR::tout && cnt == 8)) return;      // the transposed store is a warp-cooperative exchange: every lane takes part
        const long long g0 = gbase + (long long)r0 * stride;
        if (cnt == 8) {                                     // whole group
            T o1[8], o2[8];
            if constexpr (Ring::on) {                           // t' = d + x from the ring slot of this tile, stored (not transposed)
                ring->at(r0, [&](const T* d) {
                    T* __restrict__ px = X + g0;
#pragma unroll
                    for (int u = 0; u < 8; u++) { st_stream(px, PassOp<T, OP>::out_d(xs[u], d[u]), pol); px += stride; }
                });
                return;
            } else {
                if (group_reads > 0 && valid && r0 != pf_row) fetch(r0);
#pragma unroll
                for (int u = 0; u < 8; u++) PassOp<T, OP>::out(xs[u], pb[u], pc[u], o1[u], o2[u]);
            }
            pf_row = -1;
            if (TR::tout) {
                store8_transposed<T, W>(w, r0, lane, o1, X + tbase + r0, n, nvalid, pol);
                if (TR::two_out) store8_transposed<T, W>(w, r0, lane, o2, X2 + tbase + r0, n, nvalid, pol);
            } else {
                T* __restrict__ px = X + g0;                // one pointer, bumped by the row stride
#pragma unroll
                for (int u = 0; u < 8; u++) { st_stream(px, o1[u], pol); px += stride; }
            }
            return;
        }
        for (int u = 0; u < cnt; u++) {                      // the last, partial group of a fiber
            const long long g = g0 + u * stride;
            T o1, o2;
            PassOp<T, OP>::out(xs[u], TR::drain_reads > 0 ? B[g] : T(0), TR::drain_reads > 1 ? C[g] : T(0), o1, o2);
            if (TR::tout) { const long long tg = tbase + (long long)lane * n + r0 + u; X[tg] = o1; if (TR::two_out) X2[tg] = o2; }
            else X[g] = o1;
        }
    }
    template <class Env> __device__ __forceinline__ void flush(Env&, const Window<T, W>&, int, bool) {}
    __device__ __forceinline__ int hold(int, int) const { return 0x3fffffff; }
};

// ---------------------------------------------------------------- CONTIG layout: feed and drain
// Fibers are contiguous in memory (element stride 1), 32 consecutive fibers form a group.  A TMA box = BR rows x 32 fibers with
// BR * sizeof(T) = 128 bytes, so that every fiber contributes one full 128-byte line; it is written fiber-major with the 128-byte
// hardware swizzle (16-byte chunk c of fiber j sits at chunk c ^ (j & 7)) straight into the window region of those BR rows (4 KB,
// 1 KB aligned) and transposed IN PLACE through registers: lane j reads its own fiber's 128 bytes (8 conflict-free 16-byte loads),
// the warp synchronises, lane j writes its window column.  On the way out the sweep hands each lane 8 consecutive results of its
// fiber; they go straight into a swizzled staging box (conflict-free 16-byte stores) that leaves with one TMA store per BR rows.
template <typename T, int W> struct FeedContig {
    static constexpr int R = 128 / (int)sizeof(T);          // rows per box: 16 (f64) / 32 (f32)
    static constexpr int MAXQ = W / R;
    static constexpr int NBAR = W / R;
    static constexpr int EPC = 16 / (int)sizeof(T);          // elements per 16-byte chunk
    const LaneArgs<T>* a; T* win; uint64_t* bar; int f0, q0, lane;
    template <class Env> __device__ __forceinline__ void request(Env&, int row0) {
        __syncwarp();
        if (lane == 0) {
            fence_proxy_async();
            const unsigned q = (unsigned)row0 / (unsigned)R - (unsigned)q0;
            uint64_t* b = bar + (q % (unsigned)NBAR);
            mbar_expect_tx(b, 4096u);
            tma_load_3d(win + ((row0 & (W - 1)) << 5), &a->tmA, row0, f0, 0, b);
        }
    }
    template <class Env> __device__ __forceinline__ bool landed(Env&, int row0, bool block) {
        const unsigned q = (unsigned)row0 / (unsigned)R - (unsigned)q0;
        uint64_t* b = bar + (q % (unsigned)NBAR);
        const uint32_t parity = (uint32_t)((q / (unsigned)NBAR) & 1u);
        bool ok = __all_sync(0xffffffffu, mbar_test(b, parity));
        if (!ok && !block) return false;
        while (!ok) ok = __all_sync(0xffffffffu, mbar_try(b, parity));
        // in-place transpose of the 4 KB region: [fiber][row] swizzled  ->  [row][fiber]
        T* reg = win + ((row0 & (W - 1)) << 5);
        const uint32_t src = s32(reg) + (uint32_t)lane * 128u;
        T v[R];
#pragma unroll
        for (int c = 0; c < 8; c++) Vec16<T>::ld(src + (uint32_t)((c ^ (lane & 7)) << 4), v + c * EPC);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < R; i++) reg[i * LANES + lane] = v[i];
        __syncwarp();
        return true;
    }
};

template <typename T, int W> struct DrainContig {
    static constexpr int R = 128 / (int)sizeof(T);
    static constexpr int EPC = 16 / (int)sizeof(T);
    const LaneArgs<T>* a; T* stg; int f0, lane, ce;
    // xs: results of rows r0 .. r0+7 of this lane's fiber (r0 % 8 == 0); rows beyond the fiber are clipped by the TMA store
    __device__ __forceinline__ void rows8(const Window<T, W>&, int r0, int cnt, int, const T* xs, bool) {
        const int off = r0 & (R - 1);
        if (off == 0) { if (lane == 0) bulk_wait_read<0>(); __syncwarp(); }      // the previous box has left the staging tile
        const uint32_t dst = s32(stg) + (uint32_t)lane * 128u;
        const int c0 = off / EPC;
#pragma unroll
        for (int c = 0; c < 8 / EPC; c++) Vec16<T>::st(dst + (uint32_t)(((c0 + c) ^ (lane & 7)) << 4), xs + c * EPC);
        if (off + 8 == R || r0 + cnt >= ce) {                                  // box complete (or the chunk ends inside it)
            __syncwarp();
            if (lane == 0) { fence_proxy_async(); tma_store_3d(&a->tmX, stg, r0 - off, f0, 0); bulk_commit(); }
        }
    }
    __device__ __forceinline__ void prefetch(int, int, bool) {}
    template <class Env> __device__ __forceinline__ void flush(Env&, const Window<T, W>&, int, bool final) {
        if (final) { if (lane == 0) bulk_wait_all(); __syncwarp(); }            // results are in global memory before the records go out
    }
    __device__ __forceinline__ int hold(int, int) const { return 0x3fffffff; }
};

// ---------------------------------------------------------------- the kernel
enum LaneLayout { LAY_STRIDED = 0, LAY_CONTIG = 1 };
// Shared memory of a CTA of NW warps: [NW windows][NW staging areas][NW x (flags, barriers)][reciprocal table].  Windows first: the
// swizzled boxes of the CONTIG layout need 1 KB alignment, which the 16 / 32 KB windows and 4 KB staging boxes keep by themselves.
template <typename T, int W, int RT, int OP, int LAY, int NW> struct LaneSmem {
    static constexpr int NST = 2;
    static constexpr size_t win_bytes = (size_t)W * LANES * sizeof(T);
    static constexpr size_t stg_bytes = LAY == LAY_CONTIG ? 4096 : (OpTraits<OP>::staged ? (size_t)2 * NST * RT * LANES * sizeof(T) : 0);
    static constexpr size_t flg_bytes = ((size_t)LANES * (W + 8) + 127) / 128 * 128;
    static constexpr size_t bar_bytes = 128;            // W / RT <= 16 barriers
    static constexpr size_t off_stg = (size_t)NW * win_bytes;
    static constexpr size_t off_flg = off_stg + (size_t)NW * stg_bytes;
    static constexpr size_t off_rcp = off_flg + (size_t)NW * (flg_bytes + bar_bytes);
    static constexpr size_t total = off_rcp + ((W + 2) * sizeof(acc_t) + 15) / 16 * 16;
};

// repair of ONE fiber: exact sequential continuation from the last verified renewal state (verify_repair_fiber).  Executed by all
// 32 lanes of the warp redundantly and in lock step (same records, same decisions), so that the staging can be cooperative: before
// each repair scan the lanes copy the next NB rows of the fiber -- with the pass's input arithmetic applied -- into the warp's
// window memory, and the scan reads them from there (a dependent global load per step would cost ~1 us each); rows beyond the
// staged range fall back to global memory.  Lane 0 writes the results.  Rare: a handful of fibers per solve.
template <typename T, int OP, int NB, int W, bool LAMF = false>
__device__ __noinline__ int repair_fiber(const LaneArgs<T>* a, const ChunkPlan pl, long long fiber, long long gbase, long long stride, long long tfib,
                                         long long nfp, T* buf, const acc_t* rcp, int lane) {
    const int* rec = a->rec;
    const long long cstride = (long long)a->plan.nmax;
    const T* A = a->A; const T* B = a->B; const T* C = a->C; T* X = a->X; T* X2 = a->X2;
    int buf_lo = 0, buf_n = 0;
    auto in_at = [&](int r) { const long long g = gbase + (long long)r * stride;
                              return OpTraits<OP>::staged ? PassOp<T, OP>::in(A[g], B[g], C[g]) : A[g]; };
    // 256 rows are staged at a time (a repair usually merges after a few rows; staging costs up to three dependent global loads per row)
    constexpr int NBS = NB < 256 ? NB : 256;
    auto stage = [&](int pos) { __syncwarp();
                                buf_lo = pos; buf_n = pl.n - pos < NBS ? pl.n - pos : NBS;
                                for (int j = lane; j < buf_n; j += 32) buf[j] = in_at(pos + j);
                                __syncwarp(); };
    // LAMF: record index fiber = group * LANES + lane of a group (slab z, first column x0) is fiber z inc + x0 + lane
    const long long grp = fiber / LANES;
    return verify_repair_fiber<T>(pl, LAMF ? fiber_lam<T>(*a, (grp / a->gps) * a->inc + (grp % a->gps) * LANES + fiber % LANES) : a->lam,
        [&](int c) { return rec[(0 * cstride + c) * nfp + fiber]; },
        [&](int c) { return rec[(3 * cstride + c) * nfp + fiber]; },
        [&](int c) { return rec[(4 * cstride + c) * nfp + fiber]; },
        [&](int c) { return rec[(1 * cstride + c) * nfp + fiber]; },
        [&](int c) { return rec[(2 * cstride + c) * nfp + fiber]; },
        [&](int pos) { stage(pos); },
        [&](int r) { if (r < buf_lo || r >= buf_lo + buf_n) stage(r);        // warp-uniform: all lanes run the same scan
                     return buf[r - buf_lo]; },
        [&](int r, T v) { if (lane == 0) { const long long g = gbase + (long long)r * stride;
                                           T o1, o2;
                                           PassOp<T, OP>::out(v, OpTraits<OP>::drain_reads > 0 ? B[g] : T(0), OpTraits<OP>::drain_reads > 1 ? C[g] : T(0), o1, o2);
                                           if (OpTraits<OP>::tout) { X[tfib + r] = o1; if (OpTraits<OP>::two_out) X2[tfib + r] = o2; }
                                           else X[g] = o1; } },
        rcp, W + 2);
}

__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ unsigned smid() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }

// Residency the register allocation is held to: 12 warps per SM (three CTAs of 4 warps: at most 168 registers per thread), except
// for the staged forms, whose 8 KB of operand staging per warp leave room for 8 warps only (two CTAs: up to 255 registers -- the d
// ring of LOP_DR_B lives in what the third CTA would have used).
template <int OP, int NW> constexpr int lane_min_ctas() { return ((OpTraits<OP>::staged ? 8 : 12) + NW - 1) / NW; }

// LAMF: per-fiber penalties (plain op): each lane reads its fiber's penalty once, at task start, and uses it for the scan, the tail and
// the repair of its fiber; a CONTIG warp's 32 fibers may belong to two penalty groups, a STRIDED warp's lie in one slab.
template <typename T, int W, int RT, int TITER, int OP, int NW, int LAY, bool LOG, bool LAMF = false>
__global__ void __launch_bounds__(NW * 32, lane_min_ctas<OP, NW>()) k_lane(const __grid_constant__ LaneArgs<T> a) {
    using SM = LaneSmem<T, W, RT, OP, LAY, NW>;
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    acc_t* rcp = reinterpret_cast<acc_t*>(smem + SM::off_rcp);
    T* win = reinterpret_cast<T*>(smem + (size_t)warp * SM::win_bytes);
    T* stB = reinterpret_cast<T*>(smem + SM::off_stg + (size_t)warp * SM::stg_bytes);
    T* stC = stB + (LAY == LAY_CONTIG ? 0 : SM::NST * RT * LANES);
    uint8_t* flg = smem + SM::off_flg + (size_t)warp * (SM::flg_bytes + SM::bar_bytes);
    uint64_t* bar = reinterpret_cast<uint64_t*>(flg + SM::flg_bytes);

    for (int k = threadIdx.x; k < W + 2; k += NW * 32) rcp[k] = k ? 1.0 / (acc_t)k : 0.0;
    const long long task = (long long)blockIdx.x * NW + warp;
    const bool has_task = task < a.ntasks;
    if (has_task) {
        if (lane < W / RT) mbar_init(bar + lane, 1);
        for (int k = lane; k < (int)(SM::flg_bytes / 4); k += 32) reinterpret_cast<uint32_t*>(flg)[k] = 0u;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();                                    // the only CTA barrier: reciprocal table ready
    if (!has_task) return;
    // task log (tools: the LOG instantiation, launched only when a.tlog is set), TLOG_WORDS words per task:
    //   [0] start ns  [1] scan end ns  [2] end ns (globaltimer)  [3] SM id  [4] epochs  [5] scan steps  [6] starved epochs (< DMIN steps)
    //   [7] tile waits  [8] cycles in the epoch loop (clock64), of which  [9] blocked on a tile  [10] rest of nobody-can-move (tail,
    //   retirement)  [11] sweep + drain  [12] feed (requests, landing)  [13] scan  (the remainder: the epoch's warp reductions)
    //   [14] rows the task scans (owned + halo)  [15] 0
    unsigned long long* const tl = LOG ? a.tlog + task * TLOG_WORDS : nullptr;
    if (tl && lane == 0) { tl[0] = gtimer(); tl[3] = smid(); }
    struct TLogEnd { unsigned long long* p; __device__ ~TLogEnd() { if (p) *p = gtimer(); } } tlog_end{tl && lane == 0 ? tl + 2 : nullptr};

    long long group; int chunk, nc;
    a.plan.locate(task, &group, &chunk, &nc);
    const ChunkPlan pl = a.plan.plan(nc);
    const int z = (int)(group / a.gps);
    const int x0 = (int)(group - (long long)z * a.gps) * LANES;
    const TaskGeom g = pl.geom(chunk);
    const bool valid = (long long)x0 + lane < a.per_slab;
    // element (row 0) of this lane's fiber, and its element stride
    const long long gbase = LAY == LAY_CONTIG ? ((long long)x0 + lane) * pl.n : (long long)z * a.inc * pl.n + x0 + lane;
    const long long gstride = LAY == LAY_CONTIG ? 1 : a.inc;
    const long long tgroup = ((long long)z * a.inc + x0) * pl.n;      // transposed results: (fiber 0 of the group, row 0)
    const long long nfp = (long long)a.slabs * a.gps * LANES;
    const long long fiber = group * LANES + lane;

    // LAMF: this lane's penalty (an invalid lane takes lane 0's)
    const T lamf = LAMF ? fiber_lam<T>(a, (long long)z * a.inc + x0 + (valid ? lane : 0)) : T(0);
    DevEnv<T, W, LAMF> env; env.lane = lane; env.lamc = a.lamc;
    env.dw.wbase = s32(win); env.dw.lane8 = lane * (uint32_t)sizeof(T); env.dw.flg = s32(flg) + lane * (uint32_t)Window<T, W>::FP; env.dw.rcp = s32(rcp);
    Window<T, W> w{win, flg};
    if constexpr (LAMF) env.L.init(w, lane, g, lamf, valid); else env.L.init(w, lane, g, a.lam, valid);
    TaskStats ts{};
    TaskStats* const sp = LOG ? &ts : nullptr;
    const long long tc0 = LOG ? clock64() : 0;
    if constexpr (LAY == LAY_CONTIG) {
        FeedContig<T, W> feed{&a, win, bar, x0, g.p0 / FeedContig<T, W>::R, lane};
        DrainContig<T, W> drain{&a, stB, x0, lane, g.ce};
        if constexpr (LAMF) warp_task<T, W, TITER>(env, feed, drain, w, rcp, g, LaneLam<T>{lamf}, TITER + TITER / 2 + FeedContig<T, W>::R, sp);
        else warp_task<T, W, TITER>(env, feed, drain, w, rcp, g, a.lam, TITER + TITER / 2 + FeedContig<T, W>::R, sp);
    } else {
        DRing<T, W, OP> ring;
        FeedStrided<T, W, RT, OP> feed{&a, win, stB, stC, bar, x0, z, g.p0 / RT, lane, &ring};
        DrainStrided<T, W, OP> drain; drain.ring = &ring; drain.B = a.B; drain.C = a.C; drain.X = a.X; drain.X2 = a.X2; drain.gbase = gbase; drain.stride = a.inc;
        drain.pf_row = -1; drain.pol = policy_evict_first(); drain.ce = g.ce; drain.tbase = tgroup; drain.n = pl.n; drain.nvalid = (int)(a.per_slab - x0 < LANES ? a.per_slab - x0 : LANES);
        if constexpr (LAMF) warp_task<T, W, TITER>(env, feed, drain, w, rcp, g, LaneLam<T>{lamf}, TITER + TITER / 2 + RT, sp);
        else warp_task<T, W, TITER>(env, feed, drain, w, rcp, g, a.lam, TITER + TITER / 2 + RT, sp);
    }
    if (tl && lane == 0) {
        tl[1] = gtimer();
        tl[4] = ts.epochs; tl[5] = ts.iters; tl[6] = ts.starved; tl[7] = ts.waits; tl[8] = clock64() - tc0;
        tl[9] = ts.c_wait; tl[10] = ts.c_stuck; tl[11] = ts.c_sweep; tl[12] = ts.c_feed; tl[13] = ts.c_scan; tl[14] = g.ce - g.p0; tl[15] = 0;
    }

    // ---- chunk records; the last warp of the fiber group to finish verifies (and repairs) its 32 fibers ----
    int* rec = a.rec;
    const long long cstride = (long long)a.plan.nmax;
    rec[(0 * cstride + chunk) * nfp + fiber] = env.L.in_rec;
    rec[(1 * cstride + chunk) * nfp + fiber] = env.L.out_rec;
    rec[(2 * cstride + chunk) * nfp + fiber] = env.L.retired ? env.L.ovf_rec : REC_NONE;
    rec[(3 * cstride + chunk) * nfp + fiber] = env.L.in_rec2;
    rec[(4 * cstride + chunk) * nfp + fiber] = env.L.in_rec3;
    const bool any_retired = __any_sync(0xffffffffu, env.L.retired);
    if (nc == 1 && !any_retired) return;
    __threadfence();
    __syncwarp();
    int old = 0;
    if (lane == 0) old = atomicAdd(a.group_count + group, 1);
    old = __shfl_sync(0xffffffffu, old, 0);
    if (old != nc - 1) return;
    __threadfence();
    if (lane == 0) a.group_count[group] = 0;
    // quick test first: every entry record equals the predecessor's exit record and nobody retired
    bool bad = false;
    if (valid) {
        for (int c = 0; c < nc; c++) {
            const int ri = __ldcg(rec + (0 * cstride + c) * nfp + fiber);
            const int ro = c > 0 ? __ldcg(rec + (1 * cstride + c - 1) * nfp + fiber) : ri;
            const int rv = __ldcg(rec + (2 * cstride + c) * nfp + fiber);
            bad |= (c > 0 && ri != ro) || rv != REC_NONE;
        }
    }
    // the fibers that need it are repaired one after the other, by the whole warp (see repair_fiber)
    unsigned m = __ballot_sync(0xffffffffu, bad);
    int nrep = 0;
    while (m) {
        const int src = __ffs(m) - 1; m &= m - 1;
        const long long gb = __shfl_sync(0xffffffffu, gbase, src);
        nrep += repair_fiber<T, OP, W * LANES, W, LAMF>(&a, pl, group * LANES + src, gb, gstride, tgroup + (long long)src * pl.n, nfp, win, rcp, lane);
    }
    if (nrep && lane == 0) atomicAdd(a.stats, (unsigned long long)nrep);
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr; cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 3D view (d0 contiguous) of `base`; box (b0, b1, 1)
template <typename T>
static bool make_map(CUtensorMap* m, const T* base, long long d0, long long d1, long long d2, int b0, int b1, CUtensorMapSwizzle sw) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
    cuuint64_t strides[2] = {(cuuint64_t)d0 * sizeof(T), (cuuint64_t)d0 * (cuuint64_t)d1 * sizeof(T)};
    cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, 1};
    cuuint32_t es[3] = {1, 1, 1};
    const CUtensorMapDataType dt = sizeof(T) == 8 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    return fn(m, dt, 3, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct LaneTuning { int clen, halo, variant; };
static int env_variant() { const char* e = getenv("PTV_LANE_VARIANT"); return e ? atoi(e) : -1; }
static LaneTuning g_tune = {0, 32, env_variant()};        // chunk length (0 = one wave), halo rows, variant (-1: default per storage type; tools: PTV_LANE_VARIANT)
static unsigned long long* g_tlog = nullptr; static long long g_tlog_cap = 0;
void lane_set_tasklog(unsigned long long* dev, long long cap_tasks) { g_tlog = dev; g_tlog_cap = cap_tasks; }
void lane_set_tuning(int clen, int halo, int variant) { g_tune.clen = clen; g_tune.halo = halo; g_tune.variant = variant; }

// Scratch of the lane engine, one buffer per device (grow-only, zero-initialised when (re)allocated):
//     [stats 64 B][group counters: cap_groups ints][chunk records: 5 per (chunk, fiber)]
// The counters must be zero between launches (the last warp of a group resets its counter), so their region has a FIXED size per
// allocation -- it must never overlap what an earlier launch with fewer groups used for records.  A launch bakes the split (records
// at group_count + cap_groups) into its arguments, and a regrown buffer may come back at the same address with a larger counter
// region: `gen` counts the allocations, so that a captured graph can tell a stale layout from the current one (solver.cu: DrGraphKey).
struct LaneScratch { void* p = nullptr; size_t cap = 0; long long cap_groups = 0; unsigned long long gen = 0; };
static LaneScratch g_scr[ptv::MAX_DEVICES];
static long long lane_scratch_bytes(long long groups_cap, long long nf, int len) {
    const long long nfp = (nf + 31) / 32 * 32 + 32 * 64;
    const long long maxchunks = len / 64 + 2;
    return 64 + groups_cap * 4 + 5 * maxchunks * nfp * 4 + 256;
}

// launch one instantiation; with `slots` only report how many warp tasks the device can hold at once
template <typename T, int W, int RT, int TITER, int OP, int NW, int LAY, bool LAMF = false>
static cudaError_t launch_v(LaneArgs<T>& a, cudaStream_t st, int* slots) {
    using SM = LaneSmem<T, W, RT, OP, LAY, NW>;
    auto kern = k_lane<T, W, RT, TITER, OP, NW, LAY, false, LAMF>;
    const size_t smem = SM::total;
    static int s_slots = 0;                      // per instantiation: resident warps on the current device
    if (!s_slots) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NW * 32, smem);
        if (e != cudaSuccess) return e;
        s_slots = sms * per_sm * NW;
    }
    if (slots) { *slots = s_slots; return cudaSuccess; }
    const unsigned blocks = (unsigned)((a.ntasks + NW - 1) / NW);
    if constexpr (!LAMF) {
        if (a.tlog) {                            // tools: the instrumented copy (same shared memory, same residency)
            auto klog = k_lane<T, W, RT, TITER, OP, NW, LAY, true>;
            cudaError_t e = cudaFuncSetAttribute(klog, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            cudaFuncSetAttribute(klog, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            klog<<<blocks, NW * 32, smem, st>>>(a);
            return cudaGetLastError();
        }
    }
    kern<<<blocks, NW * 32, smem, st>>>(a);
    return cudaGetLastError();
}

// tuning variants (window rows, warps per CTA); 0 is the default: CTAs of 4 warps -- one per SM sub-partition -- three of which fit
// an SM when the pass needs no staging (12 resident warps, 3 per sub-partition; single-warp CTAs only reach 11, unevenly spread)
template <typename T, int OP, int LAY, bool LAMF = false>
static cudaError_t launch_variant(int variant, LaneArgs<T>& a, cudaStream_t st, int* slots) {
    if constexpr (LAMF) {           // per-fiber penalties: the default variant of each storage type only (lane_prox picks 6 / 0)
        if constexpr (sizeof(T) == 4) return launch_v<T, 128, 8, 32, OP, 4, LAY, true>(a, st, slots);
        else return launch_v<T, 64, 8, 16, OP, 4, LAY, true>(a, st, slots);
    }
    switch (variant) {
        case 1: return launch_v<T, 64, 8, 16, OP, 1, LAY>(a, st, slots);
        case 5: return launch_v<T, 128, 8, 16, OP, 1, LAY>(a, st, slots);
        case 6: if constexpr (sizeof(T) == 4) return launch_v<T, 128, 8, 32, OP, 4, LAY>(a, st, slots);      // float32: same bytes, twice the rows, half the epochs
                else return launch_v<T, 64, 8, 16, OP, 4, LAY>(a, st, slots);
        case 7: return launch_v<T, 64, 8, 24, OP, 4, LAY>(a, st, slots);      // 24-step epochs: -1 % on config 2, but only 20 window rows of slack
        default: return launch_v<T, 64, 8, 16, OP, 4, LAY>(a, st, slots);
    }
}
template <typename T>
static cudaError_t launch_any(int lay, int op, int variant, LaneArgs<T>& a, cudaStream_t st, int* slots) {
    if (a.lamf) return lay == LAY_CONTIG ? launch_variant<T, LOP_PLAIN, LAY_CONTIG, true>(variant, a, st, slots)
                                         : launch_variant<T, LOP_PLAIN, LAY_STRIDED, true>(variant, a, st, slots);
    if (lay == LAY_CONTIG) return launch_variant<T, LOP_PLAIN, LAY_CONTIG>(variant, a, st, slots);
    switch (op) {
        case LOP_DR_B: return launch_variant<T, LOP_DR_B, LAY_STRIDED>(variant, a, st, slots);
        case LOP_DR_B_FINAL: return launch_variant<T, LOP_DR_B_FINAL, LAY_STRIDED>(variant, a, st, slots);
        case LOP_DRA: return launch_variant<T, LOP_DRA, LAY_STRIDED>(variant, a, st, slots);
        case LOP_DRA_FINAL: return launch_variant<T, LOP_DRA_FINAL, LAY_STRIDED>(variant, a, st, slots);
        case LOP_DRB: return launch_variant<T, LOP_DRB, LAY_STRIDED>(variant, a, st, slots);
        case LOP_PLAIN_T: return launch_variant<T, LOP_PLAIN_T, LAY_STRIDED>(variant, a, st, slots);
        default: return launch_variant<T, LOP_PLAIN, LAY_STRIDED>(variant, a, st, slots);
    }
}

// x = prox_{lam TV}(in) over the fibers (nf, len, inc) of an array (the reference's slicing rule, src/TVNDopt.cpp:184-188).
//   inc > 1: STRIDED layout, any op (PassOp);   inc == 1: CONTIG layout, plain op only.
//   ops that write transposed (LANE_DRA, LANE_DRA_FINAL, LANE_DRB, LANE_PLAIN_T): X (and X2) are fiber-major arrays, element (fiber f, row r) at
//   f * len + r -- for the fibers of a 2D image that is the transposed image.
// scratch: lane_scratch() (records, group counters).  Returns cudaErrorInvalidConfiguration when the shape does not suit TMA
// tiling (unaligned base, row pitch not a multiple of 16 bytes, tiny fibers) -- the caller then uses the chunked engine.
// lamf (plain op only): fiber j's penalty is lamf[j / fpi] (device table, every entry > 0: the caller's to ensure), lam unused.
template <typename T>
cudaError_t lane_prox(int op, const T* A, const T* B, const T* C, T* X, long long nf, int len, long long inc, T lam, void* scratch,
                      cudaStream_t st, T* X2, const T* lamf, long long fpi) {
    if (lamf && (op != LOP_PLAIN || fpi < 1)) return cudaErrorInvalidConfiguration;
    if (nf <= 0 || len < 2 || !(lamf || lam > T(0)) || op < 0 || op > LOP_PLAIN_T) return cudaErrorInvalidConfiguration;
    const int lay = inc == 1 ? LAY_CONTIG : LAY_STRIDED;
    if (lay == LAY_CONTIG && op != LOP_PLAIN) return cudaErrorInvalidConfiguration;
    if (lay == LAY_STRIDED && nf % inc != 0) return cudaErrorInvalidConfiguration;
    const bool staged = op == LOP_DR_B || op == LOP_DR_B_FINAL, tout = op >= LOP_DRA;
    const long long pitch = (lay == LAY_CONTIG ? (long long)len : inc) * (long long)sizeof(T);
    if (pitch % 16 != 0 || ((uintptr_t)A & 15) || ((uintptr_t)X & 15) || (B && ((uintptr_t)B & 15)) || (C && ((uintptr_t)C & 15)))
        return cudaErrorInvalidConfiguration;
    if (tout && (((long long)len * (long long)sizeof(T)) % 16 != 0 || (op == LOP_DRA && (!X2 || ((uintptr_t)X2 & 15))))) return cudaErrorInvalidConfiguration;
    LaneArgs<T> a;
    memset(&a, 0, sizeof(a));
    a.A = A; a.B = B; a.C = C; a.X = X; a.X2 = X2; a.lam = lam; a.lamc[0] = 2.0 * (acc_t)lam; a.lamc[1] = -a.lamc[0];
    a.lamf = lamf; a.fpi = fpi;
    const int BR = 128 / (int)sizeof(T);
    if (lay == LAY_CONTIG) {
        if (nf > 0x7fffffff) return cudaErrorInvalidConfiguration;
        if (!make_map<T>(&a.tmA, A, len, nf, 1, BR, LANES, CU_TENSOR_MAP_SWIZZLE_128B)) return cudaErrorInvalidConfiguration;
        if (!make_map<T>(&a.tmX, X, len, nf, 1, BR, LANES, CU_TENSOR_MAP_SWIZZLE_128B)) return cudaErrorInvalidConfiguration;
        a.inc = 1; a.per_slab = nf; a.slabs = 1; a.gps = (int)((nf + LANES - 1) / LANES);
    } else {
        const long long slabs = nf / inc;
        if (slabs > 0x7fffffff) return cudaErrorInvalidConfiguration;
        if (!make_map<T>(&a.tmA, A, inc, len, slabs, LANES, 8, CU_TENSOR_MAP_SWIZZLE_NONE)) return cudaErrorInvalidConfiguration;
        if (staged) {
            if (!make_map<T>(&a.tmB, B, inc, len, slabs, LANES, 8, CU_TENSOR_MAP_SWIZZLE_NONE)) return cudaErrorInvalidConfiguration;
            if (!make_map<T>(&a.tmC, C, inc, len, slabs, LANES, 8, CU_TENSOR_MAP_SWIZZLE_NONE)) return cudaErrorInvalidConfiguration;
        }
        a.inc = inc; a.per_slab = inc; a.slabs = (int)slabs; a.gps = (int)((inc + LANES - 1) / LANES);
    }
    // Chunking.  Enough fiber groups to fill the device's resident warp slots (a batch of images, a volume): whole fibers, one warp
    // task per group (on an H100, 132 SMs x 12 warps = 1584 slots); splitting fibers into chunks there only adds halo work, and a
    // partial second wave is cheap because the SMs it leaves half empty run their warps faster.  Fewer groups
    // (one image: 128): as many chunks per fiber as fit ONE wave, floor(slots / groups), each scanned by its own warp from a cold
    // start `halo` rows early; chunk boundaries balance owned rows + halo and fall on the feed's tile rows: 8 (STRIDED), 16 / 32
    // (CONTIG) (ChunkPlan).  More chunks than that -- e.g. 13 x 128 = 1664 tasks for 1584 slots -- would put the excess into a
    // second wave a whole task long.
    const long long groups = (long long)a.slabs * a.gps;
    int slots = 0;
    const int variant = g_tune.variant >= 0 ? g_tune.variant : (sizeof(T) == 4 ? 6 : 0);      // float32: 128-row window, 32-step epochs
    cudaError_t e = launch_any<T>(lay, op, variant, a, st, &slots);
    if (e != cudaSuccess) return e;
    const int gran = lay == LAY_CONTIG ? BR : 8;
    const int halo = (g_tune.halo + gran - 1) / gran * gran;
    const int cmax = ChunkPlan::fit(len, len / 64 > 0 ? len / 64 : 1, halo, gran);      // chunks own at least ~64 rows
    a.plan.n = len; a.plan.halo = halo; a.plan.gran = gran; a.plan.gfull = groups;
    if (g_tune.clen > 0) {                                       // tools: fixed chunk length
        const int nc = (len + g_tune.clen - 1) / g_tune.clen;
        a.plan.nmax = nc < cmax ? nc : cmax;
    } else if (groups >= slots) a.plan.nmax = 1;
    else { const long long c = slots / groups; a.plan.nmax = c < cmax ? (int)c : cmax; }
    if (a.plan.nmax < 1) a.plan.nmax = 1;
    if (a.plan.nmax > len / 64 + 2) return cudaErrorInvalidConfiguration;
    {
        const int d = ptv::device_slot();
        if (d < 0 || scratch != g_scr[d].p || groups > g_scr[d].cap_groups) return cudaErrorInvalidValue;      // not lane_scratch()'s buffer
        a.stats = (unsigned long long*)scratch;
        a.group_count = (int*)((char*)scratch + 64);
        a.rec = a.group_count + g_scr[d].cap_groups;
    }
    a.ntasks = a.plan.ntasks(groups);
    a.tlog = (g_tlog && a.ntasks <= g_tlog_cap) ? g_tlog : nullptr;
    return launch_any<T>(lay, op, variant, a, st, nullptr);
}

bool lane_shape_ok(long long nf, int len, long long inc, size_t elem, const void* const* ptrs, int nptrs) {
    if (nf <= 0 || len < 2) return false;
    if (inc > 1 && nf % inc != 0) return false;
    const long long pitch = (inc == 1 ? (long long)len : inc) * (long long)elem;
    if (pitch % 16 != 0) return false;
    for (int i = 0; i < nptrs; i++) if (ptrs[i] && ((uintptr_t)ptrs[i] & 15)) return false;
    return encode_fn() != nullptr;
}

void* lane_scratch(long long nf, int len) {
    const int d = ptv::device_slot();
    if (d < 0) return nullptr;
    LaneScratch& s = g_scr[d];
    const long long groups = nf + 64;                   // upper bound on the fiber groups of any slicing of nf fibers
    const long long gcap = groups > s.cap_groups ? groups : s.cap_groups;
    const size_t need = (size_t)lane_scratch_bytes(gcap, nf, len);
    if (need > s.cap || groups > s.cap_groups) {
        if (s.p) { cudaDeviceSynchronize(); cudaFree(s.p); s.p = nullptr; s.cap = 0; }
        if (cudaMalloc(&s.p, need) != cudaSuccess) { cudaGetLastError(); s.p = nullptr; s.cap_groups = 0; return nullptr; }
        cudaMemset(s.p, 0, need); s.cap = need; s.cap_groups = gcap; s.gen++;
    }
    return s.p;
}
unsigned long long lane_scratch_generation() {
    const int d = ptv::device_slot();
    return d < 0 ? 0 : g_scr[d].gen;
}
unsigned long long lane_read_stats(int reset) {
    const int d = ptv::device_slot();
    if (d < 0 || !g_scr[d].p) return 0;
    unsigned long long v = 0;
    cudaDeviceSynchronize();
    cudaMemcpy(&v, g_scr[d].p, sizeof(v), cudaMemcpyDeviceToHost);
    if (reset) cudaMemset(g_scr[d].p, 0, sizeof(v));
    return v;
}

template cudaError_t lane_prox<double>(int, const double*, const double*, const double*, double*, long long, int, long long, double, void*, cudaStream_t, double*,
                                       const double*, long long);
template cudaError_t lane_prox<float>(int, const float*, const float*, const float*, float*, long long, int, long long, float, void*, cudaStream_t, float*,
                                      const float*, long long);

}  // namespace ptvl
