/* libxsmm_b200 -- the utility layer the reference's drivers are written against: wall-clock timer, matrix
 * comparison (libxsmm_matdiff and its scalar verdict), the sequence generator, low-precision array
 * conversions, and the handful of helper macros the samples use.
 *
 * Replaces the declarations of the reference's include/libxsmm_utils.h (-> include/utils/libxsmm_timer.h:22-42,
 * include/libxsmm_math.h:101-160, include/utils/libxsmm_math.h:17-31, include/utils/libxsmm_lpflt_quant.h:45-59)
 * and the macros of include/libxsmm_macros.h that samples/hello/hello.c, samples/xgemm_sparse/spmm_kernel.c and
 * samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c use. Same names, argument order and meaning; the
 * implementations live in libxsmm_b200/csrc/host_utils.c and are host code (nothing here touches the GPU).
 */
#ifndef LIBXSMM_UTILS_H
#define LIBXSMM_UTILS_H

/* the reference headers bring these in (include/libxsmm_macros.h); its samples rely on that */
#include <assert.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "libxsmm_macros.h"
#include "libxsmm_typedefs.h"

#if defined(__cplusplus)
extern "C" {
#endif

/* ---- element type -> datatype enumerator: LIBXSMM_DATATYPE(double) == LIBXSMM_DATATYPE_F64 ------------------- */
#define LIBXSMM_TYPESYMBOL_double F64
#define LIBXSMM_TYPESYMBOL_float F32
#define LIBXSMM_TYPESYMBOL_int I32
#define LIBXSMM_TYPESYMBOL_short I16
#define LIBXSMM_TYPESYMBOL_libxsmm_bfloat16 BF16
#define LIBXSMM_TYPESYMBOL_libxsmm_float16 F16
#define LIBXSMM_TYPESYMBOL(TYPE) LIBXSMM_CONCATENATE(LIBXSMM_TYPESYMBOL_, TYPE)
#define LIBXSMM_DATATYPE(TYPE) LIBXSMM_CONCATENATE(LIBXSMM_DATATYPE_, LIBXSMM_TYPESYMBOL(TYPE))

/* ---- seeded deterministic fill used by the drivers (reference include/libxsmm_math.h:17-56) ---------------
 * SEED != 0: element (row j, col i) = (SEED*SCALE + SCALE) * (1 + i*NROWS + j), padding rows = SEED;
 * SEED == 0: values spread over [-SCALE, +SCALE] by a coprime stride over the LD x NCOLS index space. */
#define LIBXSMM_MATINIT(TYPE, SEED, DST, NROWS, NCOLS, LD, SCALE) do { \
  const double xb_mi_seed_ = (double)(SEED), xb_mi_scale_ = xb_mi_seed_ * (SCALE) + (SCALE); \
  const libxsmm_blasint xb_mi_nr_ = (libxsmm_blasint)(NROWS), xb_mi_nc_ = (libxsmm_blasint)(NCOLS), xb_mi_ld_ = (libxsmm_blasint)(LD); \
  libxsmm_blasint xb_mi_c_, xb_mi_r_; \
  if (0 != xb_mi_seed_) { \
    for (xb_mi_c_ = 0; xb_mi_c_ < xb_mi_nc_; ++xb_mi_c_) { \
      for (xb_mi_r_ = 0; xb_mi_r_ < xb_mi_ld_; ++xb_mi_r_) { \
        ((TYPE*)(DST))[xb_mi_c_ * xb_mi_ld_ + xb_mi_r_] = (xb_mi_r_ < xb_mi_nr_) \
          ? (TYPE)(xb_mi_scale_ * (1.0 + (double)xb_mi_c_ * xb_mi_nr_ + xb_mi_r_)) : (TYPE)xb_mi_seed_; \
      } \
    } \
  } else { \
    const libxsmm_blasint xb_mi_total_ = xb_mi_nc_ * xb_mi_ld_; \
    const TYPE xb_mi_half_ = (TYPE)((libxsmm_blasint)LIBXSMM_UPDIV(xb_mi_total_, 2)); \
    const TYPE xb_mi_inv_ = ((TYPE)(SCALE)) / xb_mi_half_; \
    const size_t xb_mi_stride_ = libxsmm_coprime2((size_t)xb_mi_total_); \
    for (xb_mi_c_ = 0; xb_mi_c_ < xb_mi_total_; ++xb_mi_c_) { \
      ((TYPE*)(DST))[xb_mi_c_] = xb_mi_inv_ * ((TYPE)(xb_mi_stride_ * xb_mi_c_ % xb_mi_total_) - xb_mi_half_); \
    } \
  } \
} while (0)

/* ---- two values sharing storage (reference include/libxsmm_typedefs.h:181-189) ------------------------------ */
typedef union libxsmm_bfloat16_f32 { libxsmm_bfloat16 i[2]; float f; } libxsmm_bfloat16_f32;
typedef union libxsmm_bfloat8_f16 { libxsmm_bfloat8 i[2]; libxsmm_float16 hf; } libxsmm_bfloat8_f16;

/* ---- timer (reference include/utils/libxsmm_timer.h:22-42) --------------------------------------------------- */
typedef struct libxsmm_timer_info { int tsc; } libxsmm_timer_info;
LIBXSMM_API int libxsmm_get_timer_info(libxsmm_timer_info* info);
LIBXSMM_API libxsmm_timer_tickint libxsmm_timer_tick(void);                 /* monotonic, nanosecond ticks */
LIBXSMM_API double libxsmm_timer_duration(libxsmm_timer_tickint tick0, libxsmm_timer_tickint tick1);   /* seconds */
static inline libxsmm_timer_tickint libxsmm_timer_ncycles(libxsmm_timer_tickint tick0, libxsmm_timer_tickint tick1) {
  return LIBXSMM_DELTA(tick0, tick1);
}

/* ---- matrix comparison (reference include/libxsmm_math.h:101-160, src/libxsmm_math.c:35-447) ------------------
 * column-major m x n matrices `ref` and `tst` with leading dimensions *ldref / *ldtst (NULL: m). Field for field
 * the reference's structure: norms per http://www.netlib.org/lapack/lug/node75.html, Kahan-compensated sums. */
typedef struct libxsmm_matdiff_info {
  double norm1_abs, norm1_rel;       /* one-norm (max column sum) of the difference, relative to the reference's */
  double normi_abs, normi_rel;       /* infinity-norm (max row sum) */
  double normf_rel;                  /* Frobenius norm of the difference relative to the reference's */
  double linf_abs, linf_rel, l2_abs, l2_rel, rsq;
  double l1_ref, min_ref, max_ref, avg_ref, var_ref;
  double l1_tst, min_tst, max_tst, avg_tst, var_tst;
  double v_ref, v_tst;               /* the two values at the location of linf_abs */
  libxsmm_blasint m, n, i, r;        /* location (row m, column n) of linf_abs; i/r: bookkeeping of matdiff_reduce */
} libxsmm_matdiff_info;
LIBXSMM_API int libxsmm_matdiff(libxsmm_matdiff_info* info, libxsmm_datatype datatype, libxsmm_blasint m, libxsmm_blasint n,
  const void* ref, const void* tst, const libxsmm_blasint* ldref, const libxsmm_blasint* ldtst);
LIBXSMM_API double libxsmm_matdiff_epsilon(const libxsmm_matdiff_info* input);   /* the scalar the drivers threshold */
LIBXSMM_API void libxsmm_matdiff_reduce(libxsmm_matdiff_info* output, const libxsmm_matdiff_info* input);
LIBXSMM_API void libxsmm_matdiff_clear(libxsmm_matdiff_info* info);

/* ---- small math helpers (reference include/libxsmm_math.h:163-200) --------------------------------------------- */
LIBXSMM_API size_t libxsmm_coprime(size_t n, size_t minco);    /* a co-prime of n that is <= minco (1 if none) */
LIBXSMM_API size_t libxsmm_coprime2(size_t n);                 /* a co-prime of n close to sqrt(n) */
LIBXSMM_API double libxsmm_dsqrt(double x);
LIBXSMM_API float libxsmm_ssqrt(float x);

/* ---- sequence generator (reference include/utils/libxsmm_math.h:17-31, src/libxsmm_rng.c): xoshiro128+ in 16 lanes -- */
/* small math helpers of the reference's utility library (include/utils/libxsmm_math.h:54, include/libxsmm_math.h:267) */
LIBXSMM_API float libxsmm_sexp2_i8(signed char x);      /* 2^x */
LIBXSMM_API float libxsmm_sexp2_i8i(int x);             /* 2^x, -128 <= x <= 127 */
LIBXSMM_API float libxsmm_nearbyintf(float x);
LIBXSMM_API double libxsmm_nearbyint(double x);
LIBXSMM_API void libxsmm_rng_set_seed(unsigned int seed);
/* caller-owned generator state for DROPOUT / STOCHASTIC_ROUND kernels: 4 x 16 words, lane l seeded like libxsmm_rng_set_seed
 * (reference include/libxsmm_math.h:222-231, src/libxsmm_rng.c:172-210) */
LIBXSMM_API unsigned int* libxsmm_rng_create_extstate(unsigned int seed);
LIBXSMM_API unsigned int libxsmm_rng_get_extstate_size(void);
LIBXSMM_API void libxsmm_rng_destroy_extstate(unsigned int* stateptr);
LIBXSMM_API void libxsmm_rng_f32_seq(float* rngs, libxsmm_blasint count);     /* uniform in [0, 1) */
LIBXSMM_API unsigned int libxsmm_rng_u32(unsigned int n);                       /* uniform in [0, n) */
LIBXSMM_API void libxsmm_rng_seq(void* data, size_t nbytes);
LIBXSMM_API double libxsmm_rng_f64(void);                                       /* uniform in [0, 1) */

/* ---- low-precision array conversions (reference include/utils/libxsmm_lpflt_quant.h:45-59) ------------------- */
LIBXSMM_API void libxsmm_truncate_convert_f32_bf16(const float* in, libxsmm_bfloat16* out, size_t length);
LIBXSMM_API void libxsmm_rnaz_convert_fp32_bf16(const float* in, libxsmm_bfloat16* out, size_t length);
LIBXSMM_API void libxsmm_rne_convert_fp32_bf16(const float* in, libxsmm_bfloat16* out, size_t length);
LIBXSMM_API void libxsmm_convert_bf16_f32(const libxsmm_bfloat16* in, float* out, size_t length);
LIBXSMM_API void libxsmm_rne_convert_fp32_f16(const float* in, libxsmm_float16* out, size_t length);
LIBXSMM_API void libxsmm_convert_f16_f32(const libxsmm_float16* in, float* out, size_t length);
LIBXSMM_API void libxsmm_rne_convert_fp32_bf8(const float* in, libxsmm_bfloat8* out, size_t length);
/* stochastic rounding with the 16-lane generator state (reference src/libxsmm_lpflt_quant.c:332-368) */
LIBXSMM_API void libxsmm_stochastic_convert_fp32_bf8(const float* in, libxsmm_bfloat8* out, unsigned int len, void* rng_state, unsigned int start_seed_idx);
LIBXSMM_API void libxsmm_convert_bf8_f32(const libxsmm_bfloat8* in, float* out, size_t length);
LIBXSMM_API void libxsmm_rne_convert_fp32_hf8(const float* in, libxsmm_hfloat8* out, size_t length);
LIBXSMM_API void libxsmm_convert_hf8_f32(const libxsmm_hfloat8* in, float* out, size_t length);

/* ---- target queries (reference include/libxsmm_cpuid.h:80-120) ----------------------------------------------------
 * libxsmm_cpuid: this backend's single target, ordered above every x86 id (see LIBXSMM_B200_SM90A above).
 * libxsmm_cpuid_dot_pack_factor: elements of a k-group in the "VNNI" operand layouts the kernels consume:
 * 2 for 16-bit types, 4 for 8-bit types, else 1 -- the x86 convention (src/libxsmm_cpuid_x86.c), which IS the ABI. */
typedef struct libxsmm_cpuid_info { char model[1024]; int constant_tsc; int has_context; } libxsmm_cpuid_info;
LIBXSMM_API int libxsmm_cpuid(libxsmm_cpuid_info* info);
LIBXSMM_API int libxsmm_cpuid_dot_pack_factor(libxsmm_datatype datatype);
LIBXSMM_API int libxsmm_cpuid_vlen32(int id);
/* case-insensitive strstr (reference include/libxsmm_memory.h) */
LIBXSMM_API const char* libxsmm_stristr(const char a[], const char b[]);

#if defined(__cplusplus)
}
#endif
#endif /* LIBXSMM_UTILS_H */
