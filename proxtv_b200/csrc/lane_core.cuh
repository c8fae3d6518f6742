// lane_core.cuh -- the lane-per-fiber streaming engine of the exact 1D TV-L1 prox (host+device: the same source runs in the
// CUDA kernel, kernels_lane.cu, and lane by lane on the CPU, tests/emu/emu_lane.cu).
//
// What it computes: x = argmin 1/2 |x - y|^2 + lam * sum |x_i - x_{i+1}| for every fiber -- the minimiser the reference
// obtains with src/TVL1opt_hybridtautstring.cpp:56-235 (== src/TVL1opt.cpp:359-564, linearized taut string).  The scan is the
// same taut-string walk (same break decisions, same backtracking to the last touch point, same closing rule with the 1e-10
// tolerance at the last sample, :176,:201), but carried in SLOPE FORM: instead of the heights of the two candidate lines over
// the tube centre, updated incrementally (`mnHeight += mn - y[i]`, :84), it keeps the cumulative sum S since the anchor of
// the current segment and compares slopes,
//        cl = (S - lam - A) / k      slope from the anchor to the tube floor at sample i     (A = anchor height, k = i - last)
//        ch = (S + lam - A) / k      slope from the anchor to the tube ceiling
//        ceiling violation  <=>  lo > ch        floor violation  <=>  hi < cl        touches:  lo = max(lo, cl), hi = min(hi, ch)
// which is the same mathematics with 8 instead of 20 float64 operations per step and no division (k is a small integer: a table
// of correctly rounded reciprocals).  Results agree with the reference to a few ulp (not bit for bit: the rounding sequence
// differs), jump sets are identical away from exact ties; the bit-faithful kernels (kernels_chunked.cu) remain the ones behind
// the 1D entry points.  With Z = S - lam - A the anchor only sets the initial Z of a segment: fiber start -lam, after a
// ceiling break 0, after a floor break -2 lam -- the scan state after a break is a pure function of (position, kind), the
// renewal property (SURVEY.md 0.7) that makes speculative starts exact once they meet the true scan.
//
// GPU mapping.  One LANE owns one fiber (or one chunk of it), a warp owns 32 ADJACENT fibers, and the samples stream through a
// circular shared-memory window laid out [row = sample][lane = fiber]: lane j only ever touches column j, so every shared
// access of the scan is bank-conflict free no matter how far the lanes' positions diverge, warps never wait for each other
// (no CTA barrier in the scan), and for fibers that are adjacent in memory (every dimension but the first of a column-major
// array) a window row is one contiguous 256-byte line -- the strided pass needs no transpose at all.  Finished segments
// leave their value at their first row (the slot is dead by then) plus a one-byte flag; a lock-step sweep expands them
// and hands finished rows to the drain.  Long fibers (one image = only 4096 fibers) are cut into chunks of a few hundred
// samples that start cold `halo` samples early; a chunk is exact iff the (start, kind) of its segment covering its first row
// equals the predecessor's record of the same segment, which the last warp of a fiber group to finish verifies; a mismatch
// (or a segment too long for the window) is repaired by an exact sequential continuation from the last verified renewal state,
// which stops as soon as it reproduces one of the chunk's recorded segment starts (its first three): a few rows, as a rule.
#pragma once
#include <type_traits>
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#ifndef PTV_HD
#define PTV_HD __host__ __device__ __forceinline__
#endif

namespace ptvl {

constexpr int LANES = 32;
enum : int { LK_CEIL = 0, LK_FLOOR = 1, LK_BEGIN = 2 };          // kind of a segment start (how its anchor was set)
constexpr int REC_NONE = -1;                                     // record: no valid (start, kind)
PTV_HD int rec_pack(int pos, int kind) { return pos * 4 + kind; }
PTV_HD int rec_pos(int r) { return r >> 2; }
PTV_HD int rec_kind(int r) { return r & 3; }

// All scan arithmetic is carried in float64 whatever the storage type: a float32 array is read, accumulated and compared in
// double and only the results are rounded to float32 (the reference itself upcasts float32 input, prox_tv/__init__.py:118-121).
typedef double acc_t;
PTV_HD acc_t z_of_kind(int kind, acc_t lam) { return kind == LK_CEIL ? 0.0 : (kind == LK_FLOOR ? -2.0 * lam : -lam); }

// ------------------------------------------------------------------------------------------------------------------
// Exact sequential scan in slope form from a renewal state, generic over how samples are read and results written.
// Used by the repair path of the kernel (global memory), the tail of a fiber (window) and the CPU tests.
//   ld(i)              sample i of the fiber
//   seg(f, e, v, kind) called for every finished segment [f, e] with value v whose start has `kind`; returns true to stop
//   rcp[0 .. nrcp)     optional table of reciprocals 1 / k (the kernel's shared-memory table)
// Starts at position `pos` with a segment of kind `kind` beginning there; runs to the end of the fiber (n) unless stopped.
template <typename T, class Ld, class Seg>
PTV_HD void slope_seq(int n, T lam_, int pos, int kind, Ld ld, Seg seg, const acc_t* rcp = nullptr, int nrcp = 0) {
    const acc_t lam = (acc_t)lam_, lam2 = 2.0 * lam, eps = 1e-10;      // src/general.h:64
    int last = pos - 1, i = pos, blo = pos, bhi = pos, kcur = kind;
    acc_t Z = z_of_kind(kind, lam), lo = 0.0, hi = 0.0;
    while (i < n) {
        const acc_t y = (acc_t)ld(i);
        const int k = i - last;
        const acc_t r = k < nrcp ? rcp[k] : 1.0 / (acc_t)k;      // the table holds the correctly rounded quotients: same value
        // same expressions, same association as the lanes' loop (Lane::run): identical decisions and values bit for bit
        const acc_t cl = (Z + y) * r, ch = (Z + (y + lam2)) * r;
        Z += y;
        if (i < n - 1) {
            if (k == 1) { lo = cl; hi = ch; blo = bhi = i; i++; continue; }
            if (lo > ch) {                                   // ceiling violation (hybridtautstring.cpp:93-111)
                if (seg(last + 1, blo, (T)lo, kcur)) return;
                last = blo; i = blo + 1; Z = 0.0; kcur = LK_CEIL; continue;
            }
            if (hi < cl) {                                   // floor violation (:119-137)
                if (seg(last + 1, bhi, (T)hi, kcur)) return;
                last = bhi; i = bhi + 1; Z = -lam2; kcur = LK_FLOOR; continue;
            }
            if (cl >= lo) { lo = cl; blo = i; }              // (:153-160)
            if (ch <= hi) { hi = ch; bhi = i; }              // (:143-150)
            i++;
        } else {                                             // last sample: the tube closes on its centre (:169-224)
            const acc_t c = Z + lam;
            if (k == 1) { seg(last + 1, i, (T)c, kcur); return; }
            const acc_t hl = lo * (acc_t)k - c, hh = hi * (acc_t)k - c;
            if (hl > eps) {
                if (seg(last + 1, blo, (T)lo, kcur)) return;
                last = blo; i = blo + 1; Z = 0.0; kcur = LK_CEIL; continue;
            }
            if (hh < -eps) {
                if (seg(last + 1, bhi, (T)hi, kcur)) return;
                last = bhi; i = bhi + 1; Z = -lam2; kcur = LK_FLOOR; continue;
            }
            if (hl <= 0.0) lo = c * r;
            seg(last + 1, i, (T)lo, kcur);
            return;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Shared-memory window of one warp: W rows (power of two) of 32 samples [row][lane], and one flag byte per slot kept per
// lane ([lane][row], lane pitch W + 8 bytes: a lane's 8 consecutive flags are one aligned 8-byte word and the 32 lanes' words
// of the same row group fall into different banks).  A flag byte is 0, or kind + 1 of the segment that STARTS at that row
// (written when the break that creates the segment is taken); the segment's value is stored at the same row when it is finished.
template <typename T, int W> struct Window {
    static constexpr int FP = W + 8;       // flag pitch per lane (bytes): 8-byte aligned rows, 18-word lane stride spreads the banks
    T* win;            // [W][32]
    uint8_t* flg;      // [32][FP]
    PTV_HD T ld(int row, int lane) const { return win[((row & (W - 1)) << 5) + lane]; }
    PTV_HD void st(int row, int lane, T v) const { win[((row & (W - 1)) << 5) + lane] = v; }
    // 8 consecutive rows starting at an aligned row (row0 % 8 == 0): never wraps inside the group -> one base, fixed offsets
    PTV_HD void ld8(int row0, int lane, T* t) const {
        const T* p = win + ((row0 & (W - 1)) << 5) + lane;
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = p[u * LANES];
    }
    PTV_HD void set_flag(int row, int lane, int f) const { flg[lane * FP + (row & (W - 1))] = (uint8_t)f; }
    PTV_HD int flag(int row, int lane) const { return flg[lane * FP + (row & (W - 1))]; }
    // the 8 flags of the aligned row group that starts at row0 (row0 % 8 == 0), and clearing them
    PTV_HD unsigned long long flags8(int row0, int lane) const {
        return *reinterpret_cast<const unsigned long long*>(flg + lane * FP + (row0 & (W - 1)));
    }
    PTV_HD void clear8(int row0, int lane) const { *reinterpret_cast<unsigned long long*>(flg + lane * FP + (row0 & (W - 1))) = 0ull; }
    static constexpr size_t flag_bytes() { return (size_t)LANES * FP; }
};

// What one warp task covers: rows [cs, ce) of 32 adjacent fibers of length n, entered with a cold start at p0 <= cs.
// cs and p0 are multiples of 8 (the sweep and the feed work on aligned groups of 8 rows).
struct TaskGeom {
    int n;          // samples per fiber
    int cs, ce;     // rows this task owns (ce == n: the chunk ends the fiber)
    int p0;         // cold-start row (0: the true start of the fiber)
};

// Scan state of one lane.  The kind of every segment start lives in the window's flag bytes, so the loop carries positions only.
template <typename T> struct Lane {
    acc_t Z, lo, hi;
    int i, last, blo, bhi;
    int in_rec, out_rec;  // (start, kind) of the first emitted segment / of the finished segment that covers row ce
    int in_rec2, in_rec3; // (start, kind) of the next two segment starts after the first emitted one (found by the sweep): merge points
                          // that let a repair stop after a few rows instead of a whole chunk
    bool done;            // finished (or retired); nothing more to scan
    bool valid;           // the lane has a fiber
    bool retired;         // gave up: a segment did not fit the window; ovf_rec = renewal state to continue from
    int ovf_rec;
    T xcur;               // value carried by the sweep

    template <int W>
    PTV_HD void init(const Window<T, W>& w, int lane, const TaskGeom& g, T lam, bool is_valid) {
        i = g.p0; last = g.p0 - 1; blo = bhi = g.p0;
        Z = -(acc_t)lam; lo = hi = 0.0;
        in_rec = out_rec = ovf_rec = in_rec2 = in_rec3 = REC_NONE;
        valid = is_valid; done = !is_valid; retired = false; xcur = T(0);
        w.set_flag(g.p0, lane, LK_BEGIN + 1);           // the (cold) start of the scan is a segment start of kind BEGIN
    }

    // `niter` scan steps, no bounds checks: the caller guarantees i + niter <= frontier (and <= n - 1: the last sample is never
    // processed here).  Straight-line and branch-free by design -- every lane of a warp executes the same instructions whether it
    // advances, touches or breaks (a break is a handful of selects plus predicated stores), so the lanes of a warp never diverge.
    // Once the segment that covers row ce is finished (last >= ce) the epoch loop retires the lane (settle); whatever it did beyond
    // that segment in the same call -- more breaks, more start marks, all above ce -- is never looked at.  PH1: the lane may still be in front of its first owned segment (clip to cs, record the entry state).
    template <bool PH1, int W>
    PTV_HD void run(const Window<T, W>& w, int lane, const TaskGeom& g, const acc_t* __restrict__ rcp, acc_t lam2, int niter) {
        acc_t Z_ = Z, lo_ = lo, hi_ = hi;
        int i_ = i, last_ = last, blo_ = blo, bhi_ = bhi, in_ = in_rec;
        const acc_t nlam2 = -lam2;
        for (int it = 0; it < niter; it++) {
            const acc_t y = (acc_t)w.ld(i_, lane);
            const int k = i_ - last_;
            const acc_t r = rcp[k];
            const acc_t cl = (Z_ + y) * r, ch = (Z_ + (y + lam2)) * r;      // slopes to the tube floor / ceiling at sample i
            Z_ += y;
            const bool first = (k == 1);
            const bool can = !first;
            const bool cbk = can & (lo_ > ch);
            const bool fbk = can & !cbk & (hi_ < cl);
            const bool brk = cbk | fbk;
            const int e = cbk ? blo_ : bhi_;
            const T v = (T)(cbk ? lo_ : hi_);
            const int f = last_ + 1;
            if (PH1) {
                if (brk & (e >= g.cs)) {
                    if (in_ == REC_NONE) in_ = rec_pack(f, w.flag(f, lane) - 1);
                    const int fe = f > g.cs ? f : g.cs;
                    w.st(fe, lane, v);
                    if (fe != f) w.set_flag(fe, lane, LK_BEGIN + 1);      // clipped: the sweep needs a start mark at cs
                }
            } else {
                if (brk) w.st(f, lane, v);
            }
            if (brk) w.set_flag(e + 1, lane, cbk ? LK_CEIL + 1 : LK_FLOOR + 1);      // the new segment: start mark + kind
            const bool tlo = first | (cl >= lo_), thi = first | (ch <= hi_);
            lo_ = tlo ? cl : lo_; blo_ = tlo ? i_ : blo_;
            hi_ = thi ? ch : hi_; bhi_ = thi ? i_ : bhi_;
            Z_ = cbk ? 0.0 : (fbk ? nlam2 : Z_);
            i_ = brk ? e + 1 : i_ + 1;
            last_ = brk ? e : last_;
        }
        Z = Z_; lo = lo_; hi = hi_; i = i_; last = last_; blo = blo_; bhi = bhi_; in_rec = in_;
    }

    // after run(): has the segment that covers row ce been finished?  Its start is the last start mark at or before ce.
    template <int W>
    PTV_HD void settle(const Window<T, W>& w, int lane, const TaskGeom& g) {
        if (done || last < g.ce) return;
        done = true;
        int r = g.ce;
        while (w.flag(r, lane) == 0) r--;                 // terminates: the segment's start lies inside the window
        const bool clipped = (r == g.cs) && in_rec != REC_NONE && rec_pos(in_rec) < g.cs;     // one segment spans the whole chunk
        out_rec = clipped ? in_rec : rec_pack(r, w.flag(r, lane) - 1);
    }

    // renewal state of the open segment (for retirement)
    template <int W> PTV_HD int open_rec(const Window<T, W>& w, int lane) const { return rec_pack(last + 1, w.flag(last + 1, lane) - 1); }

    // the fiber's last sample is inside the window and this lane waits in front of it: finish sequentially (closing rule)
    template <int W>
    PTV_HD void finish_tail(const Window<T, W>& w, int lane, const TaskGeom& g, T lam) {
        if (done) return;
        Lane<T>* self = this;
        // continue from the renewal state of the open segment: exact, and short (the open segment lies inside the window)
        slope_seq<T>(g.n, lam, last + 1, w.flag(last + 1, lane) - 1,
                     [&](int r) { return w.ld(r, lane); },
                     [&](int f, int e, T v, int k) {
                         if (e >= g.cs) {
                             if (self->in_rec == REC_NONE) self->in_rec = rec_pack(f, k);
                             const int fe = f > g.cs ? f : g.cs;
                             w.st(fe, lane, v); w.set_flag(fe, lane, k + 1);
                             if (e >= g.ce) { self->done = true; self->out_rec = rec_pack(f, k); }
                         }
                         return self->done; });
        done = true;
    }
};

// ------------------------------------------------------------------------------------------------------------------
// One warp task.  Env supplies the lanes and the warp collectives (device: registers + shuffles/votes; host: a loop), Feed
// brings rows into the window, Drain takes finished rows.
//   Env:   each(f(Lane&, lane)) ; rmin(f) ; rmax(f) ; any(f) ; sync() ; scan(L, w, lane, g, rcp, lam2, ph1, niter)
//   Feed:  R rows per tile (8) ; MAXQ tiles that may be outstanding ; request(env, row0) ; bool landed(env, row0, block)
//   Drain: prefetch(r0, ce, valid) ; rows8(w, r0, cnt, lane, xs, valid) inside each() for every aligned group of 8 owned rows, in order ; flush(env, w,
//          upto, final) ; hold(): first row the window still has to keep for it
// stats (optional; nullptr in production): counters, and on the device where the warp's cycles go (clock64; 0 on the host)
//   starved: scan epochs shorter than DMIN steps (every lane close to the landed frontier)
//   c_wait: blocked on the next tile (nobody can move) ; c_stuck: the rest of the nobody-can-move branch (tail, retirement)
//   c_sweep: sweep + drain, including the drain's operand prefetch ; c_feed: requests + landing ; c_scan: scan steps + settle
struct TaskStats { int epochs, retired, tail, iters; int starved, waits; long long c_wait, c_stuck, c_sweep, c_feed, c_scan; };
PTV_HD long long task_clock() {
#ifdef __CUDA_ARCH__
    return clock64();
#else
    return 0;
#endif
}

// lam: one penalty for every lane (a T), or per lane (a callable: lam(lane) -> that lane's penalty; Env::scan then gets 2 lam(lane))
template <typename T, int W, int TITER, class Env, class Feed, class Drain, class Lam>
PTV_HD void warp_task(Env& env, Feed& feed, Drain& drain, const Window<T, W>& w, const acc_t* __restrict__ rcp, const TaskGeom g, Lam lam,
                      int ahead, TaskStats* stats) {
    constexpr int R = Feed::R;
    constexpr int DMIN = 8;           // rows kept in front of a lane that overruns its chunk; epochs shorter than this count as starved
    constexpr bool per_lane = !std::is_arithmetic<Lam>::value;
    acc_t lam2 = 0.0;
    if constexpr (!per_lane) lam2 = 2.0 * (acc_t)lam;
    int row_lo = g.p0;                // first row still held by the window
    int row_req = g.p0;               // rows below have been requested
    int row_hi = g.p0;                // rows below are in the window, ready for the scan
    int fill_pos = g.cs;              // next owned row to sweep (multiple of 8)
    bool ph1 = true;                  // some lane has not emitted its first owned segment yet
    bool recs_open = true;            // some lane may still lack its second / third start record
    const int BIG = 0x3fffffff;
    // One epoch = sweep what is final, slide the window, ask for more rows, take over what has landed, run as many scan steps as
    // every participating lane can take without a bounds check.  Three warp reductions and one barrier poll in the steady state.
    for (int epoch = 0;; epoch++) {
        const int maxi = env.rmax([&](Lane<T>& L, int) { return L.done ? -1 : L.i; });
        const int low = env.rmin([&](Lane<T>& L, int) { return L.done ? BIG : L.last + 1; });
        const bool all_done = (low == BIG);
        long long tc = stats ? task_clock() : 0;
        // ---- sweep finished rows (aligned groups of 8), slide the window ----
        {
            int upto = low < g.ce ? low : g.ce;
            if (upto > row_hi) upto = row_hi;          // only retired lanes leave owned rows outside the window (repaired later)
            if (upto < g.ce) upto &= ~7;               // whole groups only, except at the very end of the chunk
            if (upto > fill_pos) {
                const int a = fill_pos;
                const bool need_recs = recs_open && env.any([&](Lane<T>& L, int) { return L.valid && L.in_rec3 == REC_NONE; });
                if (!need_recs) recs_open = false;
                env.each([&](Lane<T>& L, int lane) {
                    for (int r = a; r < upto; r += 8) {
                        T xs[8];
                        const int cnt = upto - r < 8 ? upto - r : 8;
                        const unsigned long long fl = w.flags8(r, lane);
                        T t[8];
                        w.ld8(r, lane, t);                                          // unconditional: straight-line, loads overlap
                        if (need_recs && L.in_rec3 == REC_NONE && fl != 0ull) {     // first groups of a chunk only
                            const int base = rec_pos(L.in_rec) > g.cs ? rec_pos(L.in_rec) : g.cs;
                            for (int u = 0; u < 8; u++) {
                                const int f8 = (int)((fl >> (8 * u)) & 0xffull);
                                if (f8 && r + u > base && r + u < g.ce) {
                                    if (L.in_rec2 == REC_NONE) L.in_rec2 = rec_pack(r + u, f8 - 1);
                                    else if (L.in_rec3 == REC_NONE) L.in_rec3 = rec_pack(r + u, f8 - 1);
                                }
                            }
                        }
#pragma unroll
                        for (int u = 0; u < 8; u++) {
                            L.xcur = ((fl >> (8 * u)) & 0xffull) ? t[u] : L.xcur;
                            xs[u] = L.xcur;
                        }
                        w.clear8(r, lane);
                        drain.rows8(w, r, cnt, lane, xs, L.valid);
                    }
                });
                fill_pos = upto;
                env.sync();
                drain.flush(env, w, fill_pos, false);
            }
            int nlo = all_done ? row_hi : low;
            if (nlo > fill_pos && fill_pos < g.ce) nlo = fill_pos;      // rows not swept yet (partial group) stay
            const int hold = drain.hold(fill_pos, g.ce);
            if (nlo > hold) nlo = hold;
            if (row_lo < g.cs) {
                // halo rows are never swept: their start marks are wiped when they leave the window (whole groups of 8),
                // before their slots are reused by owned rows
                nlo = nlo < g.cs ? (nlo & ~7) : nlo;
                const int c1 = nlo < g.cs ? nlo : g.cs;
                if (c1 > row_lo) { const int c0 = row_lo; env.each([&](Lane<T>&, int lane) { for (int r = c0; r < c1; r += 8) w.clear8(r, lane); }); }
            }
            if (nlo > row_lo) row_lo = nlo;
        }
        if (all_done) break;
        if (stats) stats->epochs = epoch + 1;
        env.each([&](Lane<T>& L, int) { drain.prefetch(fill_pos, g.ce, L.valid); });     // operands of the next group to be swept
        if (stats) { const long long t = task_clock(); stats->c_sweep += t - tc; tc = t; }
        // ---- feed: keep `ahead` rows in front of the fastest lane, never more than the window holds ----
        {
            int want = maxi + ahead;
            const int cap = g.ce + R;                                    // beyond the chunk only on demand (overrun of the last segment)
            if (want > cap) want = (maxi + DMIN + 1 > cap) ? maxi + DMIN + 1 : cap;
            if (want > g.n) want = g.n;
            while (row_req < want && row_req + R <= row_lo + W && row_req - row_hi < Feed::MAXQ * R) { feed.request(env, row_req); row_req += R; }
            while (row_hi < row_req && feed.landed(env, row_hi, false)) row_hi += R;      // take over what has landed
            // a feed with a short queue (MAXQ == 1) was blocked above by the tile it has just handed over: ask again
            if (Feed::MAXQ < 2)
                while (row_req < want && row_req + R <= row_lo + W && row_req - row_hi < Feed::MAXQ * R) { feed.request(env, row_req); row_req += R; }
        }
        if (stats) { const long long t = task_clock(); stats->c_feed += t - tc; tc = t; }
        // ---- how many steps can the lanes take?  Each lane runs up to TITER steps, as far as the landed rows reach (its own bound:
        //      a lane never passes lim), so the epoch lasts as long as the lane with the most room needs ----
        const int lim = row_hi < g.n - 1 ? row_hi : g.n - 1;
        int niter = env.rmax([&](Lane<T>& L, int) { const int d = lim - L.i; return L.done ? 0 : d; });
        {
            if (niter < 1) {             // nobody can move
                if (row_hi < row_req) {                                                                  // wait for the next tile
                    feed.landed(env, row_hi, true); row_hi += R;
                    if (stats) { stats->waits++; stats->c_wait += task_clock() - tc; }
                    continue;
                }
                // lanes that wait in front of the fiber's last sample: finish them once it is in the window
                const bool movable = env.any([&](Lane<T>& L, int) { return !L.done && L.i < g.n - 1; });
                if (!movable && row_hi >= g.n) {
                    env.each([&](Lane<T>& L, int lane) {
                        if constexpr (per_lane) L.template finish_tail<W>(w, lane, g, (T)lam(lane));
                        else L.template finish_tail<W>(w, lane, g, lam);
                    });
                    env.sync();
                    if (stats) { stats->tail++; stats->c_stuck += task_clock() - tc; }
                    continue;
                }
                // stuck: nothing pending, nothing more fits -> retire the lanes that pin the window
                const bool can_feed = (row_req < g.n) && (row_req + R <= row_lo + W) && (row_req - row_hi < Feed::MAXQ * R);
                if (!can_feed) {
                    env.each([&](Lane<T>& L, int lane_) {
                        if (!L.done && L.last + 1 == low) { L.done = true; L.retired = true; L.ovf_rec = L.template open_rec<W>(w, lane_); }
                    });
                    if (stats) stats->retired++;
                }
                if (stats) stats->c_stuck += task_clock() - tc;
                continue;
            }
        }
        if (niter > TITER) niter = TITER;
        if (stats) { if (niter < DMIN) stats->starved++; tc = task_clock(); }
        // ---- scan ----
        {
            const int lim_ = lim; const bool ph1_ = ph1;
            env.each([&](Lane<T>& L, int lane) {
                const int d = lim_ - L.i;
                if (!L.done && d >= 1) {
                    // Lane::run, or the kernel's equivalent device form
                    if constexpr (per_lane) env.scan(L, w, lane, g, rcp, 2.0 * (acc_t)lam(lane), ph1_, d < TITER ? d : TITER);
                    else env.scan(L, w, lane, g, rcp, lam2, ph1_, d < TITER ? d : TITER);
                    L.template settle<W>(w, lane, g);
                }
            });
            env.sync();
            if (ph1) ph1 = env.any([&](Lane<T>& L, int) { return !L.done && L.in_rec == REC_NONE; });
            if (stats) { stats->iters += niter; stats->c_scan += task_clock() - tc; }
        }
    }
    drain.flush(env, w, fill_pos, true);
}

// ------------------------------------------------------------------------------------------------------------------
// Chunking of the fibers of one group: nchunks chunks, each entered `halo` rows early, with balanced WORK -- a chunk scans its
// owned rows plus its halo (the first one has none), so the boundaries are b_c = c w - (c - 1) halo with w = (n + (nchunks - 1)
// halo) / nchunks, rounded down to multiples of `gran` (the feed's tile rows; a power of two, halo is a multiple of it).
struct ChunkPlan {
    int n, nchunks, halo, gran;
    PTV_HD int cs(int c) const {
        if (c <= 0) return 0;
        if (c >= nchunks) return n;
        const long long b = ((long long)c * ((long long)n + (long long)(nchunks - 1) * halo)) / nchunks - (long long)(c - 1) * halo;
        return (int)(b & ~(long long)(gran - 1));
    }
    PTV_HD int ce(int c) const { return c + 1 >= nchunks ? n : cs(c + 1); }
    PTV_HD TaskGeom geom(int c) const {
        TaskGeom g; g.n = n; g.cs = cs(c); g.ce = ce(c);
        g.p0 = g.cs - halo > 0 ? g.cs - halo : 0;
        return g;
    }
    // largest chunk count <= want for which every chunk owns at least 2 gran rows more than its halo costs
    static PTV_HD int fit(int n, int want, int halo, int gran) {
        int nc = want < 1 ? 1 : want;
        while (nc > 1 && ((long long)n + (long long)(nc - 1) * halo) / nc - halo < 2 * gran) nc--;
        return nc;
    }
};

// Tasks of one launch: `groups` fiber groups; the first gfull of them are cut into nmax chunks, the others into nmax - 1, so that
// the number of warp tasks can equal the number of resident warp slots of the device exactly (one balanced wave).
struct TaskPlan {
    int n, halo, gran, nmax;
    long long gfull;
    PTV_HD long long ntasks(long long groups) const { return gfull * nmax + (groups - gfull) * (nmax - 1); }
    PTV_HD void locate(long long task, long long* group, int* chunk, int* nc) const {
        const long long tf = gfull * nmax;
        if (task < tf) { *group = task / nmax; *chunk = (int)(task - *group * nmax); *nc = nmax; }
        else { const long long t2 = task - tf; const long long g2 = t2 / (nmax - 1); *group = gfull + g2; *chunk = (int)(t2 - g2 * (nmax - 1)); *nc = nmax - 1; }
    }
    PTV_HD int chunks_of(long long group) const { return group < gfull ? nmax : nmax - 1; }
    PTV_HD ChunkPlan plan(int nc) const { ChunkPlan p; p.n = n; p.nchunks = nc; p.halo = halo; p.gran = gran; return p; }
};

// ------------------------------------------------------------------------------------------------------------------
// Verification and repair of ONE fiber after all its chunks have been scanned (run by the last warp of the fiber group to
// finish).  rin/rout/rovf(c): the chunk's records for this fiber.  A chunk is exact on entry iff the (start, kind) of its
// first emitted segment equals the predecessor's record of the segment that covers the chunk's first row (both scans are then
// in the identical renewal state from that start on).  Otherwise -- or when a lane retired inside the chunk -- the exact
// sequential scan continues from the last verified renewal state, writing results directly, until one of its finished
// segments coincides with one of the recorded segment starts of a later chunk (its first, or the two after it) or the fiber ends.
// Returns the number of repair scans.
// prep(pos): called before every repair scan with its start row (the kernel stages the fiber's rows from there into shared memory).
template <typename T, class RecIn, class RecIn2, class RecIn3, class RecOut, class RecOvf, class Prep, class Ld, class St>
PTV_HD int verify_repair_fiber(const ChunkPlan& pl, T lam, RecIn rin, RecIn2 rin2, RecIn3 rin3, RecOut rout, RecOvf rovf, Prep prep, Ld ld, St st,
                               const acc_t* rcp = nullptr, int nrcp = 0) {
    int repairs = 0, c = 0;
    bool entry_ok = true;                 // chunk c is known to be exact on entry (chunk 0; or established by a merge)
    while (c < pl.nchunks) {
        int cur = REC_NONE, cnext = c + 1;
        // when the loop arrives here through `c++`, chunk c-1 was exact to its end, so rout(c-1) is a true record
        if (!entry_ok && rin(c) != rout(c - 1)) { cur = rout(c - 1); cnext = c; }
        else if (rovf(c) != REC_NONE) cur = rovf(c);
        if (cur == REC_NONE) { c++; entry_ok = false; continue; }
        repairs++;
        int resume = pl.nchunks;
        int cs_next = pl.cs(cnext), cs_own = cnext > 0 ? pl.cs(cnext - 1) : 0;     // first rows of chunk cnext / of the chunk before it
        prep(rec_pos(cur));
        slope_seq<T>(pl.n, lam, rec_pos(cur), rec_kind(cur), ld,
                     [&](int f, int e, T v, int kind) {
                         for (int r = f; r <= e; r++) st(r, v);
                         const int rp = rec_pack(f, kind);
                         while (cnext < pl.nchunks && cs_next <= e) {          // chunk starts covered by this segment
                             if (cs_next >= f && rin(cnext) == rp) { resume = cnext; return true; }
                             cs_own = cs_next; cnext++; cs_next = pl.cs(cnext);
                         }
                         // the segment starts inside chunk cnext - 1: the same (start, kind) among that chunk's recorded starts means
                         // its lane was in this very renewal state -- everything it wrote from row f on is exact
                         const int co = cnext - 1;
                         // (a lane that retired at row p scanned nothing from p on: its marks there do not count)
                         if (co >= 0 && cs_own < f && (rin2(co) == rp || rin3(co) == rp) &&
                             (rovf(co) == REC_NONE || f < rec_pos(rovf(co)))) { resume = co; return true; }
                         return false;
                     }, rcp, nrcp);
        c = resume; entry_ok = true;      // merged into chunk `resume` (or reached the end of the fiber)
    }
    return repairs;
}

}  // namespace ptvl
