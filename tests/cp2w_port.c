/*
 * cp2w_port.c -- CPU restatement of the weighted Condat / Chambolle-Pock 2D TV-L1 prox.   ** TEST INFRASTRUCTURE ONLY **
 *
 * The checker of the weighted GPU solver in proxtv_b200/csrc/cp2.cu (proxtv_CP2W_TV_*, DESIGN.md section 15.1): tests/cp2w_port.py
 * compiles it (no FMA contraction: -ffp-contract=off) into a temporary directory and loads it; the product never uses it.  The
 * reference has no weighted primal-dual solver, so it is written from the section 15.1 contract and pinned two ways by
 * tests/test_cp2w_cpu.py: with every weight equal to lambda it is tests/cp2_port.c bit for bit, and its objective agrees with
 * DR2L1W_TV's (the oracle's port) on random problems.
 *
 * minimise 1/2 ||X - Y||^2 + sum_e W1[e] |X(i+1, j) - X(i, j)| + sum_e W2[e] |X(i, j+1) - X(i, j)|.  alg 0 Condat, 1 Chambolle-Pock
 * (no accelerated rule: it takes its step sizes from one lambda).  Y, X: M x N column-major; W1 and the dual U1: (M-1) x N
 * (differences along columns), W2 and U2: M x (N-1) (along rows), all column-major.  The iteration is cp2_port.c's with one change:
 * U1[e] is clipped to [-W1[e], W1[e]] and U2[e] to [-W2[e], W2[e]] instead of [-lambda, lambda].  Step sizes, start values
 * (X = Y, U = the differences of Y, unclipped), the stop test (sqrt(sum (Xt - X)^2 / sum X^2) > 0), maxit (<= 0: 2500),
 * info[0] = iterations run + 1 and the M == 1 / N == 1 rule (the missing term left out of D) are the same.
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define ORC_MAX_ITERS_CONDAT 2500
#define ORC_RC_OK 0
#define ORC_RC_ERROR 3

static double orc_clip(double v, double w) { return v < -w ? -w : (v > w ? w : v); }

int orc_cp2w_tv(size_t M, size_t N, const double *Y, const double *W1, const double *W2, double *X, int alg, int maxit, double *info) {
    if (alg != 0 && alg != 1) { if (info) info[2] = ORC_RC_ERROR; return 0; }
    const size_t MN = M * N, M1 = M > 0 ? M - 1 : 0, N1 = N > 0 ? N - 1 : 0;
    const double sigma = 10, tau = .9 / (sigma * 8), theta = 1.;
    double *U1 = (double *)malloc(sizeof(double) * (M1 * N + 1)), *U2 = (double *)malloc(sizeof(double) * (M * N1 + 1));
    double *Xt = (double *)malloc(sizeof(double) * (MN + 1)), *Z = (double *)malloc(sizeof(double) * (MN + 1));
    size_t i, j;
    memcpy(X, Y, sizeof(double) * MN);
    for (j = 0; j < N; j++) for (i = 0; i + 1 < M; i++) U1[i + M1 * j] = Y[i + 1 + M * j] - Y[i + M * j];
    for (j = 0; j + 1 < N; j++) for (i = 0; i < M; i++) U2[i + M * j] = Y[i + M * (j + 1)] - Y[i + M * j];
    if (maxit <= 0) maxit = ORC_MAX_ITERS_CONDAT;
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
            U1[i + M1 * j] = orc_clip(U1[i + M1 * j] + sigma * (Z[i + 1 + M * j] - Z[i + M * j]), W1[i + M1 * j]);
        for (j = 0; j + 1 < N; j++) for (i = 0; i < M; i++)
            U2[i + M * j] = orc_clip(U2[i + M * j] + sigma * (Z[i + M * (j + 1)] - Z[i + M * j]), W2[i + M * j]);
    }
    if (info) { info[0] = it; info[2] = ORC_RC_OK; }
    free(U1); free(U2); free(Xt); free(Z);
    return 1;
}
