/* A plain C caller of LIBXSMM's BLAS-style GEMM, written for this repository's tests: compiled against include/ and linked with -lxsmm,
 * like an existing caller (CP2K, samples/magazine with AUTO) that relinks. It calls libxsmm_dgemm / libxsmm_sgemm and the Fortran-77
 * symbols libxsmm_dgemm_ / libxsmm_sgemm_, which libxsmm.h does not declare (a Fortran caller binds them by name, as with the reference).
 *
 *   blas_demo reject   shapes the descriptor rejects (lda < m, m = 0): each call prints "LIBXSMM_GEMM failed" and C keeps its bytes;
 *                      nothing is launched, so this runs without a GPU
 *   blas_demo run      C (+)= op(A) op(B) on HOST buffers for every transpose pair, beta 0 and 0.5 (which accumulates like 1), alpha 3
 *                      (ignored), f64 and f32, through all four symbols, against a triple loop in the exact-order kernel's order:
 *                      prints "max_abs_diff <x>" and whether C's padding rows survived
 */
#include <libxsmm.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

void libxsmm_dgemm_(const char* transa, const char* transb, const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const double* alpha, const double* a, const libxsmm_blasint* lda, const double* b, const libxsmm_blasint* ldb,
  const double* beta, double* c, const libxsmm_blasint* ldc);
void libxsmm_sgemm_(const char* transa, const char* transb, const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const float* alpha, const float* a, const libxsmm_blasint* lda, const float* b, const libxsmm_blasint* ldb,
  const float* beta, float* c, const libxsmm_blasint* ldc);

#define SENTINEL (-1234.5)

/* C[j][i] (+)= sum_s A(i,s) B(s,j), one element at a time, s ascending: the order of the exact-order kernel */
#define TRIPLE_LOOP(T, ta, tb, beta0, m, n, k, a, lda, b, ldb, c, ldc) { int i_, j_, s_; \
  for (j_ = 0; j_ < (n); ++j_) for (i_ = 0; i_ < (m); ++i_) { T* cij = (c) + (size_t)j_ * (ldc) + i_; \
    if (beta0) *cij = 0; \
    for (s_ = 0; s_ < (k); ++s_) *cij += (ta ? (a)[(size_t)i_ * (lda) + s_] : (a)[(size_t)s_ * (lda) + i_]) \
                                      * (tb ? (b)[(size_t)s_ * (ldb) + j_] : (b)[(size_t)j_ * (ldb) + s_]); } }

static double run(int f77) {
  const libxsmm_blasint m = 37, n = 13, k = 29, ldc = 41;
  const char* trans[2] = { "N", "T" };
  double diff = 0;
  int ta, tb, bi;
  for (ta = 0; ta < 2; ++ta) for (tb = 0; tb < 2; ++tb) for (bi = 0; bi < 2; ++bi) {
    const libxsmm_blasint lda = (ta ? k : m) + 3, ldb = (tb ? n : k) + 2;
    const size_t na = (size_t)lda * (ta ? m : k), nb = (size_t)ldb * (tb ? k : n), nc = (size_t)ldc * n;
    const double dalpha = 3, dbeta = bi ? 0.5 : 0;
    const float salpha = 3, sbeta = bi ? 0.5f : 0;
    double *da = malloc(na * sizeof(double)), *db = malloc(nb * sizeof(double)), *dc = malloc(nc * sizeof(double)), *dw = malloc(nc * sizeof(double));
    float *sa = malloc(na * sizeof(float)), *sb = malloc(nb * sizeof(float)), *sc = malloc(nc * sizeof(float)), *sw = malloc(nc * sizeof(float));
    size_t i;
    for (i = 0; i < na; ++i) { da[i] = (double)((int)((i * 7) % 23) - 11) / 7.0; sa[i] = (float)da[i]; }
    for (i = 0; i < nb; ++i) { db[i] = (double)((int)((i * 5) % 19) - 9) / 3.0; sb[i] = (float)db[i]; }
    for (i = 0; i < nc; ++i) {
      dc[i] = ((i % (size_t)ldc) < (size_t)m) ? (double)((int)(i % 17) - 8) / 5.0 : SENTINEL;
      sc[i] = (float)dc[i]; dw[i] = dc[i]; sw[i] = sc[i];
    }
    if (f77) {
      libxsmm_dgemm_(trans[ta], trans[tb], &m, &n, &k, &dalpha, da, &lda, db, &ldb, &dbeta, dc, &ldc);
      libxsmm_sgemm_(trans[ta], trans[tb], &m, &n, &k, &salpha, sa, &lda, sb, &ldb, &sbeta, sc, &ldc);
    } else {
      libxsmm_dgemm(trans[ta], trans[tb], &m, &n, &k, &dalpha, da, &lda, db, &ldb, &dbeta, dc, &ldc);
      libxsmm_sgemm(trans[ta], trans[tb], &m, &n, &k, &salpha, sa, &lda, sb, &ldb, &sbeta, sc, &ldc);
    }
    TRIPLE_LOOP(double, ta, tb, !bi, m, n, k, da, lda, db, ldb, dw, ldc);
    TRIPLE_LOOP(float, ta, tb, !bi, m, n, k, sa, lda, sb, ldb, sw, ldc);
    for (i = 0; i < nc; ++i) {
      const double e = fabs(dc[i] - dw[i]), f = fabs((double)sc[i] - (double)sw[i]);
      if (e > diff || e != e) diff = (e != e) ? INFINITY : e;
      if (f > diff || f != f) diff = (f != f) ? INFINITY : f;
      if ((i % (size_t)ldc) >= (size_t)m && (dc[i] != SENTINEL || sc[i] != (float)SENTINEL)) diff = INFINITY;
    }
    free(da); free(db); free(dc); free(dw); free(sa); free(sb); free(sc); free(sw);
  }
  return diff;
}

int main(int argc, char* argv[]) {
  if (argc > 1 && 0 == strcmp(argv[1], "run")) {
    const double diff = fmax(run(0), run(1));
    printf("max_abs_diff %.3e\n", diff);
    return (diff == 0) ? 0 : 2;      /* same operation order and no FMA contraction on either side: exact */
  } else {
    const libxsmm_blasint m = 8, n = 4, k = 4, short_ld = 4, zero = 0;
    const double one = 1;
    const float fone = 1;
    double a[64], b[64], c[64];
    float sa[64], sb[64], sc[64];
    int i;
    for (i = 0; i < 64; ++i) { a[i] = b[i] = sa[i] = sb[i] = 1; c[i] = sc[i] = 7; }
    libxsmm_dgemm("N", "N", &m, &n, &k, &one, a, &short_ld, b, NULL, &one, c, NULL);          /* lda < m */
    libxsmm_sgemm("N", "N", &m, &n, &k, &fone, sa, &short_ld, sb, NULL, &fone, sc, NULL);
    libxsmm_dgemm_("N", "N", &zero, &n, &k, &one, a, NULL, b, NULL, &one, c, NULL);           /* m = 0 */
    libxsmm_sgemm_("N", "N", &zero, &n, &k, &fone, sa, NULL, sb, NULL, &fone, sc, NULL);
    for (i = 0; i < 64; ++i) if (c[i] != 7 || sc[i] != 7) { printf("C was written\n"); return 1; }
    printf("reject ok\n");
    return 0;
  }
}
