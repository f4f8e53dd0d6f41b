/* TEST INFRASTRUCTURE -- not part of the product.
 *
 * The reference's own low-bit weight GEMM branches (libxsmm_reference_gemm, src/generator_gemm_reference_impl.c:1009-1272): I2X4 and
 * I1X8 x I8 / U8 -> I32 and MXFP4X2 x I8 -> F32 / BF16 with the block scales in a.tertiary and b.tertiary (address mode: arrays of
 * br pointers), exported as ref_gemm_lowbit from a header-only build of the UNMODIFIED reference. Same calling convention as
 * oracle_gemm_lowbit (oracle/oracle_lowbit.c). No reference source is copied: this file only #includes it from where it lies.
 * Recipe: `make ref` (oracle/_ref/libxsmm_ref_lowbit.so), loaded by tests/lowbit_ffi.py only.
 */
#include <libxsmm_source.h>
#include <string.h>

#define REF_API __attribute__((visibility("default")))

REF_API int ref_gemm_lowbit(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                            unsigned long long br, void* a, void* b, void* c, long long* offs_a, long long* offs_b, void* scf_a, void* scf_b)
{
  const libxsmm_gemm_shape shape = libxsmm_create_gemm_shape(dims[0], dims[1], dims[2], dims[3], dims[4], dims[5],
    (libxsmm_datatype)types[0], (libxsmm_datatype)types[1], (libxsmm_datatype)types[3], (libxsmm_datatype)types[2]);
  const libxsmm_gemm_batch_reduce_config cfg = libxsmm_create_gemm_batch_reduce_config(
    br_type == 1 ? LIBXSMM_GEMM_BATCH_REDUCE_ADDRESS : (br_type == 2 ? LIBXSMM_GEMM_BATCH_REDUCE_OFFSET
    : (br_type == 3 ? LIBXSMM_GEMM_BATCH_REDUCE_STRIDE : LIBXSMM_GEMM_BATCH_REDUCE_NONE)), (libxsmm_blasint)stride_a, (libxsmm_blasint)stride_b, 0);
  libxsmm_gemm_param p; unsigned long long brv = br; libxsmm_descriptor_blob blob; const libxsmm_gemm_descriptor* desc;
  libxsmm_init();
  memset(&p, 0, sizeof(p));
  p.op.tertiary = &brv; p.a.primary = a; p.b.primary = b; p.c.primary = c;
  p.a.secondary = offs_a; p.b.secondary = offs_b; p.a.tertiary = scf_a; p.b.tertiary = scf_b;
  desc = libxsmm_gemm_descriptor_init_brgemm(&blob, shape, flags, 0, cfg);
  if (desc == NULL) return 1;
  libxsmm_reference_gemm(&p, desc);
  return 0;
}
