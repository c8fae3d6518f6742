// vjp_core.cuh -- the exact backward pass (vector-Jacobian product) of the batched 1D TV-L1 prox, host+device: the same source runs
// in the CUDA kernels (vjp.cu) and on the CPU (tests/emu/emu_vjp.cu), so the CPU suite checks that chunking changes no bit.
//
// y = prox_{TV_w}(x) is piecewise constant.  Away from ties its Jacobian averages within each constant segment S = [a, b]: summing the
// stationarity condition of 0.5 |y - x|^2 + sum w_e |y_{e+1} - y_e| over S gives y_S = mean(x_S) + (w_b z_b - w_{a-1} z_{a-1}) / |S|
// with z_e = sgn(y_{e+1} - y_e).  For an upstream gradient g:
//     gx_i = mean of g over the segment of i            gw_e = z_e (gx_e - gx_{e+1}) on edges between segments, +0 on fused edges
// The contract, per fiber, T = storage type, all arithmetic in double, rounded to T once when stored:
//   1. edge e (0 <= e < len-1) is FUSED iff y[e] == y[e+1] (as stored) and its weight is > 0 (a zero-weight edge never fuses);
//   2. segments are the maximal runs of samples joined by fused edges;
//   3. s = 0.0, s = s + (double)g[i] over the segment's samples left to right, m = s / (double)count, gx[i] = (T)m;
//   4. gw[e] = (T)(sgn(y[e+1] - y[e]) * ((double)gx[e] - (double)gx[e+1])) on unfused edges, +0 on fused ones.
// Every segment's sum runs left to right whatever the split of the work, so the result is a pure function of (y, g, w).
//
// Work split.  A work ITEM is one chunk [c0, c1) of one fiber (with many fibers: the whole fiber).  Pass 1 (VjpScan) walks its
// rows once and finishes every segment that lies inside the chunk (gx, and gw of its fused edges and of the edges between two such
// segments).  A segment that crosses a chunk boundary is OPEN: the chunk leaves a record (VjpRec) with the partial sum of its open
// tail.  Pass 2 (vjp_carry_from) continues each open sum through the following chunks' heads -- in order, so the sum is the
// sequential one -- and hands the means back per chunk (VjpMeans).  This is the renewal idea of the forward engines: after its first
// segment boundary a chunk owes its predecessor nothing, and open segments are disjoint, so pass 2 runs one thread per chunk that opens
// one.  Pass 3 (vjp_fix_chunk) writes the open parts and the at most three edges per chunk that touch them.  A constant fiber is one
// segment: a single sequential chain through pass 2.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef PTV_HD
#define PTV_HD __host__ __device__ __forceinline__
#endif

namespace ptvv {

enum { VJP_OPEN_LEFT = 1 /* the chunk's first segment began in an earlier chunk */,
       VJP_OPEN_RIGHT = 2 /* its last segment continues into the next chunk */ };

struct VjpRec {              // left by pass 1 for every chunk (chunked work only)
    double s_tail;           // sum of g over [tail_start, c1), from 0.0, left to right (meaningful when the tail is open and began here)
    double m_first;          // (T-rounded) mean of the segment containing c0 when pass 1 finished it (not open-left, head_end >= 0)
    int head_end;            // first row e of the chunk that ends a segment, -1 if none
    int tail_start;          // first row of the segment containing c1 - 1
    int flags;               // VJP_OPEN_*
    int pad;
};
struct VjpMeans { double head, tail; };   // pass 2: (T-rounded) means of the open segments covering the chunk's head / tail

PTV_HD double vjp_sgn(double d) { return d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0); }

// Segmentation tape of one prox pass (what the backward needs of a forward output y, without y): two bitsets F, U over the linear
// elements of the array in storage order; bit i describes element i and its successor along the pass's fibers (the (nf, len, inc)
// slicing rule: the successor of element i is i + inc, except at the last sample of a fiber):
//     (F, U) = (1, 0) fused (rule 1 above: equal as stored, weight > 0)      (0, 1) unfused, the successor is greater
//              (0, 0) unfused, the successor is smaller; also every fiber's last sample      (1, 1) unfused and equal (zero weight): sign 0
// Each bitset is ceil(n / 32) uint32 words (bit i: word i / 32, bit i % 32), zero-padded to a multiple of 256 bytes.
PTV_HD size_t vjp_tape_set_bytes(long long n) { return ((size_t)((n + 31) / 32) * 4 + 255) & ~(size_t)255; }
PTV_HD void vjp_tape_encode(bool last, bool eq, bool gt, bool wpos, uint32_t& f, uint32_t& u) {
    f = (!last && eq) ? 1u : 0u;
    u = (!last && (gt || (eq && !wpos))) ? 1u : 0u;
}
// (F, U) bits of linear element i of y under the slicing rule (nf, len, inc) (weights: w laid out with len-1 samples per fiber, or
// the uniform penalty lam when w is NULL)
template <typename T>
PTV_HD void vjp_tape_edge(const T* y, long long i, int len, long long inc, double lam, const T* w, uint32_t& f, uint32_t& u) {
    const long long slab = i / (inc * (long long)len), in = i - slab * inc * (long long)len;
    const long long r = in / inc, c = in - r * inc;
    const bool last = r == (long long)len - 1;
    if (last) { f = 0; u = 0; return; }
    const T a = y[i], b = y[i + inc];
    const bool wpos = w ? w[slab * inc * (long long)(len - 1) + r * inc + c] > T(0) : lam > 0.0;
    vjp_tape_encode(false, b == a, b > a, wpos, f, u);
}
// element i's edge: fused? and its sign (meaningful on unfused edges that are not a fiber's last sample)
PTV_HD bool vjp_tape_fused(const uint32_t* F, const uint32_t* U, long long i) {
    return ((F[i >> 5] >> (i & 31)) & 1u) && !((U[i >> 5] >> (i & 31)) & 1u);
}
PTV_HD double vjp_tape_sgn(const uint32_t* F, const uint32_t* U, long long i) {
    const bool f = (F[i >> 5] >> (i & 31)) & 1u, u = (U[i >> 5] >> (i & 31)) & 1u;
    return u ? (f ? 0.0 : 1.0) : -1.0;
}

// Pass 1, one row at a time.  The caller feeds row i with g[i], y[i+1] (ignored at i == len-1) and whether edge i's weight is > 0.
// S: out.gx(row, value), out.gw(edge, value) (a no-op when gw is not wanted).
template <typename T> struct VjpScan {
    double s;                // running sum of the current segment
    double pm, psg;          // mean of the previous finished segment and the sign of the edge that ended it
    double m_first;
    int st;                  // first row of the current segment
    int c0, len, head_end;
    bool open_left, pend, fused_last;
    T yc;                    // y[i] as stored

    PTV_HD void begin(int c0_, int len_, T y0, bool open_left_) {
        s = 0.0; pm = 0.0; psg = 0.0; m_first = 0.0; st = c0_; c0 = c0_; len = len_; head_end = -1;
        open_left = open_left_; pend = false; fused_last = false; yc = y0;
    }
    template <class S> PTV_HD void row(int i, T gi, T yn, bool wpos, S& out) {
        const bool last = (i == len - 1);
        step(i, gi, !last && yn == yc && wpos, [&]() { return vjp_sgn((double)yn - (double)yc); }, out);
        if (!last) yc = yn;
    }
    // The same row with "fused" and the sign of the edge (called only when the edge is not fused and not the fiber's last) given by the
    // caller: row() derives them from y, the tape-driven kernels (vjp_tape_bits) from a pass's segmentation tape.
    template <class S, class SG> PTV_HD void step(int i, T gi, bool fu, SG sgn, S& out) {
        s = s + (double)gi;
        const bool last = (i == len - 1);
        if (fu) {
            out.gw(i, T(0));
        } else {
            // segment [st, i] ends here; pass 1 owns it unless it began in an earlier chunk
            const bool mine = !(open_left && st == c0);
            double mt = 0.0;
            if (mine) {
                mt = (double)(T)(s / (double)(i - st + 1));
                for (int k = st; k <= i; k++) out.gx(k, (T)mt);
                if (pend) out.gw(st - 1, (T)(psg * (pm - mt)));
                if (head_end < 0) m_first = mt;
            }
            if (head_end < 0) head_end = i;
            pend = mine && !last;           // edge i waits for the next segment's mean (never consumed at the chunk's end: pass 3)
            if (!last) { psg = sgn(); pm = mt; }
            s = 0.0; st = i + 1;
        }
        fused_last = fu;
    }
    PTV_HD void finish(VjpRec& r) const {
        r.s_tail = s; r.m_first = m_first; r.head_end = head_end; r.tail_start = st;
        r.flags = (open_left ? VJP_OPEN_LEFT : 0) | (fused_last ? VJP_OPEN_RIGHT : 0); r.pad = 0;
    }
};

// Pass 2 for chunk c of one fiber (records R[0..nc), chunks of C rows): if an open segment BEGINS in chunk c, continue its sum
// through the heads of the following chunks, in order, until it ends, and hand its mean to every chunk it covers.  Open segments
// are disjoint, so the chunks can be handled in any order (the device: one thread per chunk).  G: g(row) -> T.
// M: means(chunk) -> VjpMeans&.
template <typename T, class G, class M>
PTV_HD void vjp_carry_from(const VjpRec* R, int c, int nc, int C, int len, G g, M means) {
    const VjpRec& r = R[c];
    if (!(r.flags & VJP_OPEN_RIGHT) || ((r.flags & VJP_OPEN_LEFT) && r.head_end < 0)) return;
    double s = r.s_tail;
    int cnt = (c + 1) * C - r.tail_start;
    for (int k = c + 1; k < nc; k++) {                          // chunk k is open-left: its edge k * C - 1 is chunk k-1's last
        const int c0 = k * C, c1 = c0 + C < len ? c0 + C : len;
        const int he = R[k].head_end, e = he < 0 ? c1 - 1 : he;
        for (int i = c0; i <= e; i++) s = s + (double)g(i);
        cnt += e - c0 + 1;
        if (he >= 0) {
            const double m = (double)(T)(s / (double)cnt);
            means(c).tail = m;
            for (int j = c + 1; j < k; j++) { means(j).head = m; means(j).tail = m; }
            means(k).head = m;
            return;
        }
    }
}

// mean of the segment containing the first row of a chunk that is not open-left (needed by the previous chunk's last edge)
PTV_HD double vjp_first_mean(const VjpRec& r, const VjpMeans& m) { return r.head_end >= 0 ? r.m_first : m.tail; }

// Pass 3, one chunk: gx of its open parts, then gw of the edges pass 1 left: after an open head, before an open tail, and the chunk's
// last edge when it ends a segment (its right side is the next chunk's first segment, m_next = vjp_first_mean of that chunk).
// Y: y(row) -> T, X: gx(row) -> T (reads back what passes 1 and 3 stored in this chunk), W: wpos(edge) is not needed (unfused edges only).
// vjp_fix_chunk_sg: the same with the sign of an unfused edge given by the caller, SG: sg(edge) -> double (tape-driven kernels).
template <typename T, class S, class SG, class X>
PTV_HD void vjp_fix_chunk_sg(const VjpRec& r, const VjpMeans& mm, int c0, int c1, int len, double m_next, bool want_gw, SG sg, X gx, S& out);
template <typename T, class S, class Y, class X>
PTV_HD void vjp_fix_chunk(const VjpRec& r, const VjpMeans& mm, int c0, int c1, int len, double m_next, bool want_gw, Y y, X gx, S& out) {
    vjp_fix_chunk_sg<T>(r, mm, c0, c1, len, m_next, want_gw, [&](int e) { return vjp_sgn((double)y(e + 1) - (double)y(e)); }, gx, out);
}
template <typename T, class S, class SG, class X>
PTV_HD void vjp_fix_chunk_sg(const VjpRec& r, const VjpMeans& mm, int c0, int c1, int len, double m_next, bool want_gw, SG sg, X gx, S& out) {
    const bool ol = r.flags & VJP_OPEN_LEFT, orr = r.flags & VJP_OPEN_RIGHT;
    const bool inside = ol && r.head_end < 0;
    if (ol) { const int e = inside ? c1 - 1 : r.head_end; for (int k = c0; k <= e; k++) out.gx(k, (T)mm.head); }
    if (orr && !inside) for (int k = r.tail_start; k < c1; k++) out.gx(k, (T)mm.tail);
    if (!want_gw || inside) return;
    auto edge = [&](int e) {
        const double l = (double)gx(e), rr = (e == c1 - 1) ? m_next : (double)gx(e + 1);
        out.gw(e, (T)(sg(e) * (l - rr)));
    };
    if (ol && r.head_end < c1 - 1) edge(r.head_end);
    if (orr && r.tail_start > c0 && !(ol && r.head_end == r.tail_start - 1)) edge(r.tail_start - 1);
    if (c1 < len && !orr) edge(c1 - 1);
}

}  // namespace ptvv
