/* libxsmm_b200 -- preprocessor layer the reference's sample drivers are written against (target identifiers,
 * multi-dimensional array access, small arithmetic helpers). Same macro names, arguments and meaning as the
 * reference's include/libxsmm_macros.h:640-832 and include/libxsmm_cpuid.h:23-59 (the numeric target ids are part of
 * the API: drivers compare libxsmm_get_target_archid() against them); the formulations are this repository's own.
 */
#ifndef LIBXSMM_MACROS_H
#define LIBXSMM_MACROS_H

/* the reference's macro header pulls the C library in; its samples rely on that (PRIuPTR, FLT_MAX, M_PI, ...) */
#if !defined(_USE_MATH_DEFINES)
# define _USE_MATH_DEFINES 1
#endif
#include <assert.h>
#include <float.h>
#include <inttypes.h>
#include <limits.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#if !defined(M_PI)
# define M_PI 3.14159265358979323846
#endif

/* ---- code-generation targets of the reference (include/libxsmm_cpuid.h:23-59) ---------------------------------- */
#define LIBXSMM_TARGET_ARCH_UNKNOWN   0
#define LIBXSMM_TARGET_ARCH_GENERIC   1
#define LIBXSMM_X86_GENERIC           1002
#define LIBXSMM_X86_SSE3              1003
#define LIBXSMM_X86_SSE42             1004
#define LIBXSMM_X86_AVX               1005
#define LIBXSMM_X86_AVX2              1006
#define LIBXSMM_X86_AVX2_ADL          1007
#define LIBXSMM_X86_AVX2_SRF          1008
#define LIBXSMM_X86_AVX512_VL128_SKX  1041
#define LIBXSMM_X86_AVX512_VL256_SKX  1051
#define LIBXSMM_X86_AVX512_VL256_CLX  1052
#define LIBXSMM_X86_AVX512_VL256_CPX  1053
#define LIBXSMM_X86_AVX512_SKX        1101
#define LIBXSMM_X86_AVX512_CLX        1102
#define LIBXSMM_X86_AVX512_CPX        1103
#define LIBXSMM_X86_AVX512_SPR        1104
#define LIBXSMM_X86_AVX512_GNR        1105
#define LIBXSMM_X86_AVX512_DMR        1106
#define LIBXSMM_X86_AVX512_ACE1       1107
#define LIBXSMM_X86_ALLFEAT           1999
#define LIBXSMM_AARCH64_V81           2001
#define LIBXSMM_AARCH64_V82           2002
#define LIBXSMM_AARCH64_APPL_M1       2101
#define LIBXSMM_AARCH64_SVE128        2201
#define LIBXSMM_AARCH64_NEOV2         2202
#define LIBXSMM_AARCH64_SVE256        2301
#define LIBXSMM_AARCH64_NEOV1         2302
#define LIBXSMM_AARCH64_SVE512        2401
#define LIBXSMM_AARCH64_A64FX         2402
#define LIBXSMM_AARCH64_APPL_M4       2501
#define LIBXSMM_AARCH64_ALLFEAT       2999
#define LIBXSMM_RV64_MVL128           3001
#define LIBXSMM_RV64_MVL256           3002
#define LIBXSMM_RV64_MVL128_LMUL      3003
#define LIBXSMM_RV64_MVL256_LMUL      3004
#define LIBXSMM_RV64_ALLFEAT          3999
/* this backend's single target; ordered above every CPU id so that "at least <target>" feature tests hold */
#define LIBXSMM_B200_SM90A           100000

/* ---- token helpers ----------------------------------------------------------------------------------------------- */
#define LIBXSMM_CONCATENATE2(A, B) A##B
#define LIBXSMM_CONCATENATE(A, B) LIBXSMM_CONCATENATE2(A, B)
#define LIBXSMM_CONCATENATE3(A, B, C) LIBXSMM_CONCATENATE(LIBXSMM_CONCATENATE(A, B), C)
#define LIBXSMM_STRINGIFY2(SYMBOL) #SYMBOL
#define LIBXSMM_STRINGIFY(SYMBOL) LIBXSMM_STRINGIFY2(SYMBOL)
#define LIBXSMM_EXPAND(...) __VA_ARGS__
#define LIBXSMM_ELIDE(...)
#define LIBXSMM_PRAGMA(DIRECTIVE) _Pragma(LIBXSMM_STRINGIFY(DIRECTIVE))
#if defined(_OPENMP)
# define LIBXSMM_PRAGMA_SIMD LIBXSMM_PRAGMA(omp simd)
# define LIBXSMM_OPENMP_SIMD
#else
# define LIBXSMM_PRAGMA_SIMD
#endif
#define LIBXSMM_PRAGMA_NONTEMPORAL(...)
#define LIBXSMM_PRAGMA_VALIGNED
#define LIBXSMM_PRAGMA_LOOP_COUNT(MIN, MAX, AVG)
#define LIBXSMM_PRAGMA_UNROLL_N(N)
#define LIBXSMM_PRAGMA_UNROLL

#if !defined(LIBXSMM_INLINE)
# define LIBXSMM_INLINE static inline
#endif
#if !defined(LIBXSMM_INLINE_ALWAYS)
# define LIBXSMM_INLINE_ALWAYS static inline __attribute__((always_inline))
#endif
#if !defined(LIBXSMM_UNUSED)
# define LIBXSMM_UNUSED(VARIABLE) (void)(VARIABLE)
#endif
#define LIBXSMM_UNUSED_ARG __attribute__((unused))
#define LIBXSMM_ATTRIBUTE(A) __attribute__((A))
#define LIBXSMM_ATTRIBUTE_UNUSED __attribute__((unused))
#define LIBXSMM_RESTRICT __restrict__
#define LIBXSMM_ALIGNED(DECL, N) DECL __attribute__((aligned(N)))
#define LIBXSMM_ASSERT(EXPR) assert(EXPR)
#define LIBXSMM_EXPECT(EXPR) do { if (!(EXPR)) { assert(0); } } while (0)
#define LIBXSMM_ASSERT_MSG(EXPR, MSG) assert((EXPR) && *MSG)
#define LIBXSMM_LIKELY(EXPR) __builtin_expect(!!(EXPR), 1)
#define LIBXSMM_UNLIKELY(EXPR) __builtin_expect(!!(EXPR), 0)
#define LIBXSMM_ALIGNMENT 64
#define LIBXSMM_CACHELINE 64

/* ---- arithmetic helpers (arguments may be evaluated more than once, as in the reference) -------------------------- */
#define LIBXSMM_FEQ(A, B) ((A) == (B))
#define LIBXSMM_NEQ(A, B) ((A) != (B))
#define LIBXSMM_ISNAN(A) LIBXSMM_NEQ(A, A)
#define LIBXSMM_NOTNAN(A) LIBXSMM_FEQ(A, A)
#define LIBXSMM_ABS(A) (0 <= (A) ? (A) : -(A))
#define LIBXSMM_MIN(A, B) ((A) < (B) ? (A) : (B))
#define LIBXSMM_MAX(A, B) ((A) < (B) ? (B) : (A))
#define LIBXSMM_CLMP(VALUE, LO, HI) ((LO) < (VALUE) ? ((VALUE) <= (HI) ? (VALUE) : LIBXSMM_MIN(VALUE, HI)) : LIBXSMM_MAX(LO, VALUE))
#define LIBXSMM_DELTA(T0, T1) ((T0) < (T1) ? ((T1) - (T0)) : ((T0) - (T1)))
#define LIBXSMM_MOD(A, N) ((A) % (N))
#define LIBXSMM_MOD2(A, NPOT) ((A) & ((NPOT) - 1))
#define LIBXSMM_UPDIV(N, MULT) (((N) + ((MULT) - 1)) / (MULT))
#define LIBXSMM_UP(N, MULT) (LIBXSMM_UPDIV(N, MULT) * (MULT))
#define LIBXSMM_LO2(N, NPOT) ((N) & ~((NPOT) - 1))
#define LIBXSMM_UP2(N, NPOT) LIBXSMM_LO2((N) + ((NPOT) - 1), NPOT)
#define LIBXSMM_ISPOT(A) (0 != (A) && !((A) & ((A) - 1)))
#define LIBXSMM_SIGN(A) (0 < (A) ? (1) : (0 == (A) ? (0) : (-1)))
#define LIBXSMM_XOR(A, B) ((A) ^ (B))
#define LIBXSMM_ROUNDX(TYPE, A) ((TYPE)((long long)(0 <= (A) ? ((double)(A) + 0.5) : ((double)(A) - 0.5))))
#define LIBXSMM_ROUND(A) LIBXSMM_ROUNDX(double, A)
#define LIBXSMM_ROUNDF(A) LIBXSMM_ROUNDX(float, A)
#define LIBXSMM_EXP2(A) exp2(A)
#define LIBXSMM_EXP2F(A) exp2f(A)
#define LIBXSMM_LOG2(A) log2(A)
#define LIBXSMM_LOG2F(A) log2f(A)
#define LIBXSMM_POWF(A, B) powf(A, B)
#define LIBXSMM_POW(A, B) pow(A, B)
#define LIBXSMM_EXPF(A) expf(A)
#define LIBXSMM_LOGF(A) logf(A)
#define LIBXSMM_TANHF(A) tanhf(A)
#define LIBXSMM_SQRTF(A) sqrtf(A)
#define LIBXSMM_ERFF(A) erff(A)
#define LIBXSMM_FREXPF(A, B) frexpf(A, B)
#define LIBXSMM_FABSF(A) fabsf(A)
#define LIBXSMM_FABS(A) fabs(A)
/* flag arithmetic on enumerations without C++ complaints: (type)(a | b)   (reference include/libxsmm_macros.h:650) */
#define LIBXSMM_EOR(ENUM_TYPE, ENUM, FLAG) ((ENUM_TYPE)(((int)(ENUM)) | ((int)(FLAG))))
/* evaluate an expression whose value is deliberately dropped (reference :1006-1013) */
#define LIBXSMM_ELIDE_RESULT(TYPE, EXPR) do { TYPE libxsmm_b200_elided_ = (EXPR); LIBXSMM_UNUSED(libxsmm_b200_elided_); } while (0)
#define LIBXSMM_EXPECT_ELIDE(EXPR) LIBXSMM_ELIDE_RESULT(int, EXPR)
#define LIBXSMM_PUTENV(A) putenv(A)
/* build configuration the reference bakes into libxsmm_config.h (include/libxsmm_macros.h:17-27): kernels are always available here
 * (LIBXSMM_JIT != 0: a dispatch that fails is an error, tests/threadsafety.c:240), no default GEMM flags, no default prefetch */
#define LIBXSMM_JIT 1
#define LIBXSMM_FLAGS 0
#define LIBXSMM_PREFETCH LIBXSMM_GEMM_PREFETCH_NONE
/* mention a loop variable that only an OpenMP pragma uses (some compilers warn otherwise); nothing to do for gcc */
#define LIBXSMM_OMP_VAR(A)
/* checked narrowing casts of the reference (include/libxsmm_macros.h:231-264): here plain casts (LP64, 32-bit blasint) */
#define LIBXSMM_CAST_INT(VALUE) ((int)(VALUE))
#define LIBXSMM_CAST_UINT(VALUE) ((unsigned int)(VALUE))
#define LIBXSMM_CAST_LLONG(VALUE) ((long long)(VALUE))
#define LIBXSMM_CAST_BLASINT(VALUE) ((libxsmm_blasint)(VALUE))
#if defined(_OPENMP) && (201811 <= _OPENMP)
# define LIBXSMM_OMP_MASKED _Pragma("omp masked")
#else
# define LIBXSMM_OMP_MASKED _Pragma("omp master")
#endif
#define LIBXSMM_SNPRINTF(S, N, ...) snprintf(S, N, __VA_ARGS__)
#define LIBXSMM_PUT(ARRAY, I, V) ((ARRAY)[I] = (V))

/* ---- multi-dimensional view of a flat buffer ------------------------------------------------------------------------
 * LIBXSMM_VLA_DECL(<ndims>, <elem-type>, <name>, <pointer>, <s1>, ..., <s(ndims-1)>) declares the view,
 * LIBXSMM_VLA_ACCESS(<ndims>, <name>, <i0>, ..., <i(ndims-1)>, <s1>, ..., <s(ndims-1)>) is element (i0, ..., i(ndims-1))
 * of the row-major array whose trailing extents are s1..s(ndims-1). Here: a typed pointer and flat index arithmetic
 * (no variable-length array types), <ndims> must be a literal 1..6 as in every caller. */
#define LIBXSMM_VLA_POSTFIX _
#define LIBXSMM_VLA_DECL(NDIMS, ELEMENT_TYPE, VARIABLE_NAME, INIT_VALUE, ...) \
  ELEMENT_TYPE *const LIBXSMM_CONCATENATE(VARIABLE_NAME, LIBXSMM_VLA_POSTFIX) = (ELEMENT_TYPE*)(INIT_VALUE)
#define LIBXSMM_VLA_ACCESS(NDIMS, ARRAY, ...) \
  (LIBXSMM_CONCATENATE(ARRAY, LIBXSMM_VLA_POSTFIX)[LIBXSMM_CONCATENATE(LIBXSMM_B200_FLAT_, NDIMS)(__VA_ARGS__)])
#define LIBXSMM_B200_FLAT_1(I0, ...) ((size_t)(I0))
#define LIBXSMM_B200_FLAT_2(I0, I1, S1) ((size_t)(I0) * (size_t)(S1) + (size_t)(I1))
#define LIBXSMM_B200_FLAT_3(I0, I1, I2, S1, S2) (LIBXSMM_B200_FLAT_2(I0, I1, S1) * (size_t)(S2) + (size_t)(I2))
#define LIBXSMM_B200_FLAT_4(I0, I1, I2, I3, S1, S2, S3) (LIBXSMM_B200_FLAT_3(I0, I1, I2, S1, S2) * (size_t)(S3) + (size_t)(I3))
#define LIBXSMM_B200_FLAT_5(I0, I1, I2, I3, I4, S1, S2, S3, S4) (LIBXSMM_B200_FLAT_4(I0, I1, I2, I3, S1, S2, S3) * (size_t)(S4) + (size_t)(I4))
#define LIBXSMM_B200_FLAT_6(I0, I1, I2, I3, I4, I5, S1, S2, S3, S4, S5) (LIBXSMM_B200_FLAT_5(I0, I1, I2, I3, I4, S1, S2, S3, S4) * (size_t)(S5) + (size_t)(I5))

#endif /* LIBXSMM_MACROS_H */
