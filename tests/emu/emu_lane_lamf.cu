// emu_lane_lamf.cu -- TEST INFRASTRUCTURE: the lane engine's plain pass with one penalty per lane (per-fiber penalties: fiber j's is
// lamf[j / fpi]) run on the CPU through lane_core.cuh, with emu_lane.cu's host Env, feed and drains.  Each lane scans, finishes its tail
// and is repaired with its own fiber's penalty, as the LAMF instantiation of the kernel does; a warp's 32 fibers may belong to two
// penalty groups.  Not part of the product; built by tests/test_lane_lamf_emulation.py with g++.
#include "emu_lane.cu"

template <typename T, int W, int TITER, int RT>
static int run_lamf(const T* A, T* X, long long nf, int len, long long inc, const T* lamf, long long fpi, int clen, int halo, EmuStats* es) {
    if (nf <= 0 || len <= 0) return 0;
    const int boxed = inc == 1;                    // the kernel's CONTIG layout drains boxes, its STRIDED layout drains rows
    Op<T> op{0, A, nullptr, nullptr, X, nullptr};
    ChunkPlan pl; pl.n = len; pl.gran = boxed ? 16 : 8; pl.halo = (halo + pl.gran - 1) / pl.gran * pl.gran;
    pl.nchunks = (clen <= 0 || clen >= len) ? 1 : ChunkPlan::fit(len, (len + clen - 1) / clen, pl.halo, pl.gran);
    std::vector<T> win((size_t)W * LANES); std::vector<acc_t> rcp(W + 2);
    std::vector<unsigned long long> flg8((Window<T, W>::flag_bytes() + 7) / 8 + 1);
    uint8_t* flgp = reinterpret_cast<uint8_t*>(flg8.data());
    for (int k = 1; k < W + 2; k++) rcp[k] = 1.0 / (acc_t)k;
    const long long slabs = inc > 1 ? nf / inc : 1, per_slab = inc > 1 ? inc : nf;
    const long long gps = (per_slab + LANES - 1) / LANES;
    std::vector<int> rin((size_t)pl.nchunks * LANES), rout((size_t)pl.nchunks * LANES), rovf((size_t)pl.nchunks * LANES);
    std::vector<int> rin2((size_t)pl.nchunks * LANES), rin3((size_t)pl.nchunks * LANES);
    for (long long s = 0; s < slabs; s++)
        for (long long gidx = 0; gidx < gps; gidx++) {
            Fibers<T> fb; T lam[LANES];
            for (int l = 0; l < LANES; l++) {
                const long long jj = gidx * LANES + l;
                fb.valid[l] = jj < per_slab;
                if (inc > 1) { fb.base[l] = s * inc * len + jj; fb.stride = inc; fb.tbase[l] = (s * inc + jj) * len; }
                else { fb.base[l] = jj * (long long)len; fb.stride = 1; fb.tbase[l] = jj * (long long)len; }
                lam[l] = lamf[(s * (inc > 1 ? inc : 0) + (fb.valid[l] ? jj : gidx * LANES)) / fpi];    // fiber s inc + jj
            }
            auto lane_lam = [&](int l) { return lam[l]; };
            for (int c = 0; c < pl.nchunks; c++) {
                const TaskGeom g = pl.geom(c);
                Window<T, W> w{win.data(), flgp};
                memset(flgp, 0, Window<T, W>::flag_bytes());
                HostEnv<T> env;
                for (int l = 0; l < LANES; l++) env.L[l].init(w, l, g, lam[l], fb.valid[l]);
                long long fed = 0;
                HostFeed<T, W, RT> feed{&w, &op, &fb, len, &fed};
                TaskStats ts{0, 0, 0, 0};
                if (boxed) {
                    HostDrainBoxed<T, W, 16> drain{&op, &fb, g.cs, g.ce};
                    warp_task<T, W, TITER>(env, feed, drain, w, rcp.data(), g, lane_lam, TITER + RT, &ts);
                } else {
                    HostDrainDirect<T, W> drain{&op, &fb};
                    warp_task<T, W, TITER>(env, feed, drain, w, rcp.data(), g, lane_lam, TITER + RT, &ts);
                }
                for (int l = 0; l < LANES; l++) {
                    rin[(size_t)c * LANES + l] = env.L[l].in_rec; rout[(size_t)c * LANES + l] = env.L[l].out_rec;
                    rovf[(size_t)c * LANES + l] = env.L[l].retired ? env.L[l].ovf_rec : REC_NONE;
                    rin2[(size_t)c * LANES + l] = env.L[l].in_rec2; rin3[(size_t)c * LANES + l] = env.L[l].in_rec3;
                    if (env.L[l].retired) es->retired_lanes++;
                }
                es->tasks++; es->steps_max += ts.iters; es->epochs += ts.epochs; es->retired_events += ts.retired; es->tails += ts.tail; es->rows_fed += fed;
            }
            for (int l = 0; l < LANES; l++) {
                if (!fb.valid[l]) continue;
                const long long base = fb.base[l], st = fb.stride, tb = fb.tbase[l];
                es->repairs += verify_repair_fiber<T>(pl, lam[l],
                    [&](int c) { return rin[(size_t)c * LANES + l]; }, [&](int c) { return rin2[(size_t)c * LANES + l]; },
                    [&](int c) { return rin3[(size_t)c * LANES + l]; }, [&](int c) { return rout[(size_t)c * LANES + l]; },
                    [&](int c) { return rovf[(size_t)c * LANES + l]; }, [](int) {},
                    [&](int r) { return op.in(base + (long long)r * st); }, [&](int r, T v) { op.out(base + (long long)r * st, tb + r, v); });
            }
        }
    return 0;
}

extern "C" {
// the kernel's default configurations: float64 W=64, TITER=16; float32 W=128, TITER=32; 8-row tiles
int emu_lane_lamf_f64(const double* A, double* X, long long nf, int len, long long inc, const double* lamf, long long fpi, int clen, int halo,
                      long long* stats) {
    EmuStats es; memset(&es, 0, sizeof(es));
    const int rc = run_lamf<double, 64, 16, 8>(A, X, nf, len, inc, lamf, fpi, clen, halo, &es);
    if (stats) memcpy(stats, &es, sizeof(es));
    return rc;
}
int emu_lane_lamf_f32(const float* A, float* X, long long nf, int len, long long inc, const float* lamf, long long fpi, int clen, int halo,
                      long long* stats) {
    EmuStats es; memset(&es, 0, sizeof(es));
    const int rc = run_lamf<float, 128, 32, 8>(A, X, nf, len, inc, lamf, fpi, clen, halo, &es);
    if (stats) memcpy(stats, &es, sizeof(es));
    return rc;
}
}
