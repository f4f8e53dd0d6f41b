/* TEST INFRASTRUCTURE -- not part of the product.
 *
 * The reference's own MX fp8 GEMM (libxsmm_reference_gemm, src/generator_gemm_reference_impl.c:2620-2679) with the block scales in
 * a/b/c.tertiary, exported as ref_gemm_mx from a header-only build of the UNMODIFIED reference. Same calling convention as
 * oracle_gemm_mx (oracle/oracle_mx.c). No reference source is copied: this file only #includes it from where it lies. Recipe:
 * `make ref` (oracle/_ref/libxsmm_ref_mx.so), loaded by tests/mx_ffi.py only.
 */
#include <libxsmm_source.h>
#include <string.h>

#define REF_API __attribute__((visibility("default")))

REF_API int ref_gemm_mx(const int* dims, const int* types, unsigned int flags, int br_type, unsigned long long br,
                        void* a, void* b, void* c, void* a_s, void* b_s, void* c_s)
{
  const libxsmm_gemm_shape shape = libxsmm_create_gemm_shape(dims[0], dims[1], dims[2], dims[3], dims[4], dims[5],
    (libxsmm_datatype)types[0], (libxsmm_datatype)types[1], (libxsmm_datatype)types[3], (libxsmm_datatype)types[2]);
  const libxsmm_gemm_batch_reduce_config cfg = libxsmm_create_gemm_batch_reduce_config(
    br_type == 3 ? LIBXSMM_GEMM_BATCH_REDUCE_STRIDE : LIBXSMM_GEMM_BATCH_REDUCE_NONE,
    (libxsmm_blasint)((long long)dims[3] * dims[2]), (libxsmm_blasint)((long long)dims[4] * dims[2]), 0);
  libxsmm_gemm_param p; unsigned long long brv = br; libxsmm_descriptor_blob blob; const libxsmm_gemm_descriptor* desc;
  libxsmm_init();
  memset(&p, 0, sizeof(p));
  p.op.tertiary = &brv; p.a.primary = a; p.b.primary = b; p.c.primary = c;
  p.a.tertiary = a_s; p.b.tertiary = b_s; p.c.tertiary = c_s;
  desc = libxsmm_gemm_descriptor_init_brgemm(&blob, shape, flags, 0, cfg);
  if (desc == NULL) return 1;
  libxsmm_reference_gemm(&p, desc);
  return 0;
}
