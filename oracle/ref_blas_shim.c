/* TEST INFRASTRUCTURE -- not part of the product.
 *
 * The reference's own BLAS-style entry points, libxsmm_dgemm / libxsmm_sgemm (src/libxsmm_main.c:3933-3949, i.e. LIBXSMM_XGEMM
 * with its JIT kernel), exported under ref_blas_* names from a header-only build of the UNMODIFIED reference. The header-only build
 * keeps the reference's own symbols hidden, hence these forwards. No reference source is copied: this file only #includes it from
 * where it lies. Recipe: oracle/ref_blas.py, run by build() where the reference sources exist; the result, oracle/_ref/libxsmm_ref_blas.so,
 * is loaded by tests/test_blas_gemm.py only.
 */
#include <libxsmm_source.h>

#define REF_API __attribute__((visibility("default")))

REF_API void ref_blas_dgemm(const char* transa, const char* transb, const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const double* alpha, const double* a, const libxsmm_blasint* lda, const double* b, const libxsmm_blasint* ldb,
  const double* beta, double* c, const libxsmm_blasint* ldc)
{
  libxsmm_dgemm(transa, transb, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}

REF_API void ref_blas_sgemm(const char* transa, const char* transb, const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const float* alpha, const float* a, const libxsmm_blasint* lda, const float* b, const libxsmm_blasint* ldb,
  const float* beta, float* c, const libxsmm_blasint* ldc)
{
  libxsmm_sgemm(transa, transb, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}
