/*
 * cp2_dual_port.c -- the weighted Condat / Chambolle-Pock iteration of tests/cp2w_port.c, returning its final duals too.
 *   ** TEST INFRASTRUCTURE ONLY **
 *
 * The checker of the converged backward pass (proxtv_b200/csrc/cp2_vjp.cu, DESIGN.md section 15.2): its fused-edge rule reads the
 * final duals U1, U2, which the solver ports keep to themselves.  tests/cp2_vjp_host.py compiles this file (no FMA contraction) into a
 * temporary directory and loads it.  The arithmetic is cp2w_port.c's operation for operation, so X is bit for bit that port's result
 * (and, with every weight equal to lambda, cp2_port.c's); tests/test_cp2_vjp_cpu.py checks both.
 * Y, X: M x N column-major; W1, U1: (M-1) x N (edges along columns); W2, U2: M x (N-1) (along rows).  alg 0 Condat, 1 Chambolle-Pock.
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

static double dual_clip(double v, double w) { return v < -w ? -w : (v > w ? w : v); }

int orc_cp2w_duals(size_t M, size_t N, const double *Y, const double *W1, const double *W2, double *X, double *U1, double *U2, int alg,
                   int maxit, double *info) {
    if (alg != 0 && alg != 1) { if (info) info[2] = 3; return 0; }
    const size_t MN = M * N, M1 = M > 0 ? M - 1 : 0;
    const double sigma = 10, tau = .9 / (sigma * 8), theta = 1.;
    double *Xt = (double *)malloc(sizeof(double) * (MN + 1)), *Z = (double *)malloc(sizeof(double) * (MN + 1));
    size_t i, j;
    memcpy(X, Y, sizeof(double) * MN);
    for (j = 0; j < N; j++) for (i = 0; i + 1 < M; i++) U1[i + M1 * j] = Y[i + 1 + M * j] - Y[i + M * j];
    for (j = 0; j + 1 < N; j++) for (i = 0; i < M; i++) U2[i + M * j] = Y[i + M * (j + 1)] - Y[i + M * j];
    if (maxit <= 0) maxit = 2500;
    int it; double stop = DBL_MAX;
    for (it = 1; stop > 0 && it <= maxit; it++) {
        const double c = 1. / (1. + tau);
        for (j = 0; j < N; j++) for (i = 0; i < M; i++) {
            double a = 0, b = 0, D;
            if (M > 1) a = i == 0 ? -U1[M1 * j] : (i == M - 1 ? U1[M - 2 + M1 * j] : U1[i - 1 + M1 * j] - U1[i + M1 * j]);
            if (N > 1) b = j == 0 ? -U2[i] : (j == N - 1 ? U2[i + M * (N - 2)] : U2[i + M * (j - 1)] - U2[i + M * j]);
            D = (M > 1 && N > 1) ? a + b : (M > 1 ? a : (N > 1 ? b : 0.));
            const size_t q = i + M * j;
            Xt[q] = alg == 0 ? X[q] - tau * (X[q] - Y[q] + D) : c * (X[q] + tau * (Y[q] - D));
            Z[q] = Xt[q] + theta * (Xt[q] - X[q]);
        }
        double num = 0, den = 0;
        for (i = 0; i < MN; i++) { den += X[i] * X[i]; double d = Xt[i] - X[i]; num += d * d; }
        stop = sqrt(num / den);
        memcpy(X, Xt, sizeof(double) * MN);
        for (j = 0; j < N; j++) for (i = 0; i + 1 < M; i++)
            U1[i + M1 * j] = dual_clip(U1[i + M1 * j] + sigma * (Z[i + 1 + M * j] - Z[i + M * j]), W1[i + M1 * j]);
        for (j = 0; j + 1 < N; j++) for (i = 0; i < M; i++)
            U2[i + M * j] = dual_clip(U2[i + M * j] + sigma * (Z[i + M * (j + 1)] - Z[i + M * j]), W2[i + M * j]);
    }
    if (info) { info[0] = it; info[2] = 0; }
    free(Xt); free(Z);
    return 1;
}
