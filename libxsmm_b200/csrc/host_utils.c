/* libxsmm_b200 -- host utilities behind include/libxsmm_utils.h: timer, matrix comparison, sequence
 * generator, low-precision array conversions, target queries. Plain C, no device work.
 *
 * Reference roles: src/libxsmm_timer.c (monotonic tick + seconds), src/libxsmm_math.c:35-447 together with
 * src/libxsmm_matdiff.h (libxsmm_matdiff and its reductions), src/libxsmm_rng.c + src/libxsmm_utils.c:20-83
 * (xoshiro128+ lanes; scalar draws come from the C library's 48-bit generator), src/libxsmm_lpflt_quant.c:218-300
 * and src/libxsmm_math.c:587-830 (conversions). The drivers use libxsmm_matdiff_epsilon as THE pass/fail
 * number, so the statistics below follow the reference's definitions term by term (incl. Kahan-compensated
 * sums in the same visiting order); tests/test_host_utils.py pins them against the reference build.
 */
#if !defined(_DEFAULT_SOURCE)
# define _DEFAULT_SOURCE
#endif
#if !defined(_XOPEN_SOURCE)
# define _XOPEN_SOURCE 600
#endif
#include <ctype.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "../../include/libxsmm.h"
#include "../../include/libxsmm_utils.h"
#include "xb_device.cuh"

/* ---- timer ------------------------------------------------------------------------------------------ */
LIBXSMM_API int libxsmm_get_timer_info(libxsmm_timer_info* info) {
  if (info == NULL) return EXIT_FAILURE;
  info->tsc = 0;                      /* ticks are CLOCK_MONOTONIC nanoseconds, not a cycle counter */
  return EXIT_SUCCESS;
}

LIBXSMM_API libxsmm_timer_tickint libxsmm_timer_tick(void) {
  struct timespec t;
  clock_gettime(CLOCK_MONOTONIC, &t);
  return (libxsmm_timer_tickint)t.tv_sec * 1000000000ull + (libxsmm_timer_tickint)t.tv_nsec;
}

LIBXSMM_API double libxsmm_timer_duration(libxsmm_timer_tickint tick0, libxsmm_timer_tickint tick1) {
  return (double)LIBXSMM_DELTA(tick0, tick1) * 1e-9;
}

/* ---- small math ---------------------------------------------------------------------------------------- */
static size_t xb_gcd(size_t a, size_t b) { while (b != 0) { const size_t c = a % b; a = b; b = c; } return a; }

static unsigned int xb_isqrt_u64(unsigned long long x) {     /* floor(sqrt(x)), bit by bit from the top */
  unsigned int y = 0, bit;
  for (bit = 0x80000000u; bit != 0; bit >>= 1) { const unsigned long long t = (unsigned long long)(y | bit); if (t * t <= x) y |= bit; }
  return y;
}

/* Walks candidates d = |s - i| for i = n-1, n-1-j, ... (j: 1 for odd n, 2 for even n so that only odd distances from
 * the even/odd start s are visited) and keeps the first co-prime that is <= minco; if none qualifies, the co-prime
 * with the largest n % d seen. Same candidate order and tie rules as the reference (src/libxsmm_math.c:470-501): the
 * shuffle-initialised driver inputs depend on the exact value. */
LIBXSMM_API size_t libxsmm_coprime(size_t n, size_t minco) {
  const int odd = (int)(n & 1);
  const size_t start = odd ? (((minco > 1 ? minco : 1) - 1) | 1) : (minco & ~(size_t)1);
  const size_t step = odd ? 1 : 2;
  size_t result = (n > 1) ? 1 : 0, best_rem = 0, best = 1, i;
  for (i = (step < n) ? (n - 1) : 0; step < i; i -= step) {
    const size_t d = (start < i) ? (i - start) : (start - i);
    if (d != 0 && xb_gcd(n, d) == 1) {
      const size_t rem = n % d;
      result = d;
      if (best_rem < rem) { best_rem = rem; best = d; }
      if (d <= minco) break;
    }
  }
  if (minco < result) result = best;
  return result;
}

LIBXSMM_API size_t libxsmm_coprime2(size_t n) { return libxsmm_coprime(n, xb_isqrt_u64(n)); }
LIBXSMM_API double libxsmm_dsqrt(double x) { return sqrt(x); }
LIBXSMM_API float libxsmm_ssqrt(float x) { return sqrtf(x); }

/* ---- matrix comparison ------------------------------------------------------------------------------------ */
LIBXSMM_API void libxsmm_matdiff_clear(libxsmm_matdiff_info* info) {
  if (info == NULL) return;
  memset(info, 0, sizeof(*info));
  info->m = info->n = info->i = -1;                 /* no differing location yet */
  info->min_ref = info->min_tst = (double)INFINITY;
  info->max_ref = info->max_tst = -(double)INFINITY;
  info->rsq = (double)INFINITY;                     /* "not computed" (a valid R-squared is <= 1) */
}

typedef struct xb_kahan { double sum, comp; } xb_kahan;
static void xb_kadd(xb_kahan* k, double v) {        /* compensated summation, reference src/libxsmm_math.c:533-541 */
  const double c = v - k->comp, r = k->sum + c;
  k->comp = (r - k->sum) - c; k->sum = r;
}
static double xb_ratio(double nominator, double den_ref, double fallback) { return (den_ref > 0) ? (nominator / den_ref) : fallback; }

static double xb_elem(const void* p, size_t idx, int t) {
  switch (t) {
    case LIBXSMM_DATATYPE_F64: return ((const double*)p)[idx];
    case LIBXSMM_DATATYPE_F32: return (double)((const float*)p)[idx];
    case LIBXSMM_DATATYPE_F16: return (double)xb_f16_to_f32(((const unsigned short*)p)[idx]);
    case LIBXSMM_DATATYPE_BF16: return (double)libxsmm_convert_bf16_to_f32(((const unsigned short*)p)[idx]);
    case LIBXSMM_DATATYPE_BF8: { float f; libxsmm_convert_bf8_f32((const libxsmm_bfloat8*)p + idx, &f, 1); return (double)f; }
    case LIBXSMM_DATATYPE_HF8: { float f; libxsmm_convert_hf8_f32((const libxsmm_hfloat8*)p + idx, &f, 1); return (double)f; }
    case LIBXSMM_DATATYPE_I64: return (double)((const long long*)p)[idx];
    case LIBXSMM_DATATYPE_I32: return (double)((const int*)p)[idx];
    case LIBXSMM_DATATYPE_U32: return (double)((const unsigned int*)p)[idx];
    case LIBXSMM_DATATYPE_I16: return (double)((const short*)p)[idx];
    case LIBXSMM_DATATYPE_U16: return (double)((const unsigned short*)p)[idx];
    case LIBXSMM_DATATYPE_I8: return (double)((const signed char*)p)[idx];
    default: return (double)((const unsigned char*)p)[idx];   /* MXFP4X2 / NVFP4X2 / MXBF8 containers: compared as raw bytes */
  }
}

static int xb_matdiff_type_ok(int t) {
  switch (t) {
    case LIBXSMM_DATATYPE_F64: case LIBXSMM_DATATYPE_F32: case LIBXSMM_DATATYPE_F16: case LIBXSMM_DATATYPE_BF16: case LIBXSMM_DATATYPE_BF8:
    case LIBXSMM_DATATYPE_HF8: case LIBXSMM_DATATYPE_I64: case LIBXSMM_DATATYPE_I32: case LIBXSMM_DATATYPE_U32: case LIBXSMM_DATATYPE_I16:
    case LIBXSMM_DATATYPE_U16: case LIBXSMM_DATATYPE_I8: case LIBXSMM_DATATYPE_MXFP4X2: case LIBXSMM_DATATYPE_NVFP4X2: case LIBXSMM_DATATYPE_MXBF8: return 1;
    /* like the reference (src/libxsmm_math.c:52-223), plain U8 is not a comparable type */
    default: return 0;
  }
}

LIBXSMM_API int libxsmm_matdiff(libxsmm_matdiff_info* info, libxsmm_datatype datatype, libxsmm_blasint m, libxsmm_blasint n,
  const void* ref, const void* tst, const libxsmm_blasint* ldref, const libxsmm_blasint* ldtst)
{
  libxsmm_blasint ldr = (ldref != NULL) ? *ldref : m, ldt = (ldtst != NULL) ? *ldtst : m, rows = m, cols = n, c, r;
  int swapped = 0, nan_kind = 0;       /* nan_kind: 1 test value not finite, 2 reference value not finite */
  const size_t ntotal = (size_t)m * (size_t)n;
  const double inf = (double)INFINITY;
  xb_kahan k_l2rel = {0, 0}, k_l2abs = {0, 0}, k_fref = {0, 0}, k_ftst = {0, 0}, k_l1ref = {0, 0}, k_l1tst = {0, 0};
  double max_row_ref = 0, max_row_tst = 0, max_col_ref = 0;
  if (ref == NULL && tst != NULL) { ref = tst; tst = NULL; swapped = 1; }   /* one-sided statistics land in the *_tst fields */
  if (ref == NULL || info == NULL || m > ldr || m > ldt) return EXIT_FAILURE;
  if (!xb_matdiff_type_ok((int)datatype)) {
    static int error_once = 0;
    if (libxsmm_verbosity != 0 && 0 == error_once++) fprintf(stderr, "LIBXSMM ERROR: unsupported data-type requested!\n");
    return EXIT_FAILURE;
  }
  if (n == 1) { rows = ldr = ldt = 1; cols = m; }   /* a column vector is scanned as a row vector (standardises the norms) */
  libxsmm_matdiff_clear(info);

  /* pass 1, columns outer: extrema, L2/Frobenius sums, "row" sums per column index (infinity-norm in the reference's terms) */
  for (c = 0; c < cols && nan_kind == 0; ++c) {
    xb_kahan s_ref = {0, 0}, s_tst = {0, 0}, s_dif = {0, 0};
    for (r = 0; r < rows; ++r) {
      const double ti = (tst != NULL) ? xb_elem(tst, (size_t)c * ldt + r, (int)datatype) : 0.0;
      const double ri = xb_elem(ref, (size_t)c * ldr + r, (int)datatype);
      const double ta = fabs(ti), ra = fabs(ri);
      if (ri < info->min_ref) info->min_ref = ri;
      if (ri > info->max_ref) info->max_ref = ri;
      if (ti == ti && (inf > ta || ti == ri)) {
        const double di = (tst != NULL) ? fabs(ri - ti) : 0.0;
        const double dri = xb_ratio(di, ra, ta);
        if (ti < info->min_tst) info->min_tst = ti;
        if (ti > info->max_tst) info->max_tst = ti;
        if (info->linf_abs < di) { info->linf_abs = di; info->v_ref = ri; info->v_tst = ti; info->m = r; info->n = c; }
        if (info->linf_rel < dri) info->linf_rel = dri;
        if (inf > dri * dri) xb_kadd(&k_l2rel, dri * dri);
        xb_kadd(&s_ref, ra); xb_kadd(&s_tst, ta); xb_kadd(&s_dif, di);
        xb_kadd(&k_fref, ri * ri); xb_kadd(&k_ftst, ti * ti);
        if (inf > di * di) xb_kadd(&k_l2abs, di * di);
      } else {
        nan_kind = (ri == ri && inf > ra) ? 1 : 2;
        info->m = r; info->n = c; info->v_ref = ri; info->v_tst = ti;
        break;
      }
    }
    if (nan_kind == 0) {
      xb_kadd(&k_l1ref, s_ref.sum); xb_kadd(&k_l1tst, s_tst.sum);
      if (info->normi_abs < s_dif.sum) info->normi_abs = s_dif.sum;
      if (max_row_ref < s_ref.sum) max_row_ref = s_ref.sum;
      if (max_row_tst < s_tst.sum) max_row_tst = s_tst.sum;
    }
  }
  info->l2_rel = k_l2rel.sum; info->l2_abs = k_l2abs.sum; info->l1_ref = k_l1ref.sum; info->l1_tst = k_l1tst.sum;

  if (nan_kind == 0) {
    xb_kahan k_var_ref = {0, 0}, k_var_tst = {0, 0};
    double resrel;
    if (ntotal != 0) { info->avg_ref = info->l1_ref / (double)ntotal; info->avg_tst = info->l1_tst / (double)ntotal; }
    info->normi_rel = xb_ratio(info->normi_abs, max_row_ref, max_row_tst);
    { const double ft2 = k_ftst.sum * k_ftst.sum; info->normf_rel = xb_ratio(info->l2_abs, k_fref.sum, (ft2 < info->l2_abs) ? ft2 : info->l2_abs); }
    /* pass 2, rows outer: variances and the one-norm */
    for (r = 0; r < rows; ++r) {
      xb_kahan s_ref = {0, 0}, s_tst = {0, 0}, s_dif = {0, 0};
      for (c = 0; c < cols; ++c) {
        const double ri = xb_elem(ref, (size_t)c * ldr + r, (int)datatype);
        const double ti = (tst != NULL) ? xb_elem(tst, (size_t)c * ldt + r, (int)datatype) : 0.0;
        const double di = (tst != NULL) ? fabs(ri - ti) : 0.0;
        const double rd = ri - info->avg_ref, td = ti - info->avg_tst;
        xb_kadd(&k_var_ref, rd * rd); xb_kadd(&k_var_tst, td * td);
        xb_kadd(&s_ref, fabs(ri)); xb_kadd(&s_tst, fabs(ti)); xb_kadd(&s_dif, di);
      }
      if (info->norm1_abs < s_dif.sum) info->norm1_abs = s_dif.sum;
      if (max_col_ref < s_ref.sum) max_col_ref = s_ref.sum;
    }
    info->var_ref = k_var_ref.sum; info->var_tst = k_var_tst.sum;
    info->norm1_rel = xb_ratio(info->norm1_abs, max_col_ref, info->norm1_abs);
    resrel = xb_ratio(info->l2_abs, info->var_ref, info->l2_abs);
    info->rsq = (1.0 - resrel > 0.0) ? (1.0 - resrel) : 0.0;
    if (ntotal != 0) { info->var_ref /= (double)ntotal; info->var_tst /= (double)ntotal; }
    info->normf_rel = sqrt(info->normf_rel); info->l2_abs = sqrt(info->l2_abs); info->l2_rel = sqrt(info->l2_rel);
  } else {   /* a NaN/Inf: every difference statistic reads infinity, the offending side's statistics are invalidated */
    info->norm1_abs = info->norm1_rel = info->normi_abs = info->normi_rel = info->normf_rel = info->linf_abs = info->linf_rel
                    = info->l2_abs = info->l2_rel = inf;
    if (nan_kind == 1) { info->l1_tst = info->var_tst = inf; info->avg_tst = info->v_tst; info->min_tst = +inf; info->max_tst = -inf; }
    else { info->l1_ref = info->var_ref = inf; info->avg_ref = info->v_ref; info->min_ref = +inf; info->max_ref = -inf; }
  }
  if (n == 1) { const libxsmm_blasint t = info->m; info->m = info->n; info->n = t; }
  if (swapped) {
    info->min_tst = info->min_ref; info->min_ref = 0; info->max_tst = info->max_ref; info->max_ref = 0;
    info->avg_tst = info->avg_ref; info->avg_ref = 0; info->var_tst = info->var_ref; info->var_ref = 0;
    info->l1_tst = info->l1_ref; info->l1_ref = 0; info->v_tst = info->v_ref; info->v_ref = 0;
  }
  return EXIT_SUCCESS;
}

LIBXSMM_API double libxsmm_matdiff_epsilon(const libxsmm_matdiff_info* input) {
  /* the reference can also append the value to a log file named by LIBXSMM_MATDIFF (src/libxsmm_math.c:331-395);
   * that side channel is out of scope here, the number is identical */
  if (input == NULL) return 0;
  if (0 < input->rsq) {
    const double a = (input->normf_rel < input->linf_abs) ? input->normf_rel : input->linf_abs;
    return a / input->rsq;
  } else {
    const double a = (input->norm1_abs < input->normi_abs) ? input->norm1_abs : input->normi_abs;
    const double b = (input->linf_abs < input->l2_abs) ? input->l2_abs : input->linf_abs;
    return (a < b) ? b : a;
  }
}

LIBXSMM_API void libxsmm_matdiff_reduce(libxsmm_matdiff_info* output, const libxsmm_matdiff_info* input) {
  /* running worst case over several comparisons (reference src/libxsmm_math.c:398-447) */
  double eps_in, eps_out;
  if (output == NULL) return;
  if (input == NULL) { libxsmm_matdiff_clear(output); return; }
  eps_in = libxsmm_matdiff_epsilon(input); eps_out = libxsmm_matdiff_epsilon(output);
  if (output->linf_abs <= input->linf_abs) { output->linf_abs = input->linf_abs; output->linf_rel = input->linf_rel; }
  if (output->norm1_abs <= input->norm1_abs) { output->norm1_abs = input->norm1_abs; output->norm1_rel = input->norm1_rel; }
  if (output->normi_abs <= input->normi_abs) { output->normi_abs = input->normi_abs; output->normi_rel = input->normi_rel; }
  if (output->l2_abs <= input->l2_abs) { output->l2_abs = input->l2_abs; output->l2_rel = input->l2_rel; }
  if (output->normf_rel <= input->normf_rel) output->normf_rel = input->normf_rel;
  if (output->var_ref <= input->var_ref) output->var_ref = input->var_ref;
  if (output->var_tst <= input->var_tst) output->var_tst = input->var_tst;
  if (output->max_ref <= input->max_ref) output->max_ref = input->max_ref;
  if (output->max_tst <= input->max_tst) output->max_tst = input->max_tst;
  if (output->min_ref >= input->min_ref) output->min_ref = input->min_ref;
  if (output->min_tst >= input->min_tst) output->min_tst = input->min_tst;
  if (eps_out < eps_in) {       /* R-squared, location and values of the worst comparison so far */
    output->rsq = input->rsq;
    output->v_ref = input->v_ref; output->v_tst = input->v_tst;
    output->m = input->m; output->n = input->n; output->i = input->r;
  }
  output->avg_ref = 0.5 * (output->avg_ref + input->avg_ref); output->avg_tst = 0.5 * (output->avg_tst + input->avg_tst);
  output->l1_ref += input->l1_ref; output->l1_tst += input->l1_tst;
  ++output->r;
}

/* ---- small math helpers (reference src/libxsmm_utils.c:218-252, src/libxsmm_math.c:980-999) --------------------------------- */
LIBXSMM_API float libxsmm_sexp2_i8(signed char x) { return ldexpf(1.0f, (int)x); }
LIBXSMM_API float libxsmm_sexp2_i8i(int x) { return ldexpf(1.0f, x < -128 ? -128 : (x > 127 ? 127 : x)); }
LIBXSMM_API float libxsmm_nearbyintf(float x) { return nearbyintf(x); }
LIBXSMM_API double libxsmm_nearbyint(double x) { return nearbyint(x); }

/* ---- sequence generator ---------------------------------------------------------------------------------------- */
static unsigned int g_rng[4][16];       /* xoshiro128+ : four state words x sixteen independent lanes */
static int g_rng_seeded = 0;

static void xb_rng_step(unsigned int* s0, unsigned int* s1, unsigned int* s2, unsigned int* s3) {
  const unsigned int t = *s1 << 9;
  *s2 ^= *s0; *s3 ^= *s1; *s1 ^= *s2; *s0 ^= *s3; *s2 ^= t;
  *s3 = (*s3 << 11) | (*s3 >> 21);
}

/* lane l starts at (seed + 31-l, seed + 131-l, seed + 231-l, seed + 331-l) and is then advanced by 2^64 draws with the
 * generator's jump polynomial, so that the lanes never overlap (reference src/libxsmm_rng.c:30-106); state[w * 16 + lane] */
static void xb_rng_seed_lanes(unsigned int seed, unsigned int* state) {
  static const unsigned int jump[4] = { 0x8764000bu, 0xf542d2d3u, 0x6fa035c3u, 0x77f2db5bu };
  int lane, w, b;
  for (lane = 0; lane < 16; ++lane) {
    unsigned int s[4], acc[4] = {0, 0, 0, 0};
    for (w = 0; w < 4; ++w) s[w] = seed + (unsigned int)(100 * w + 31 - lane);
    for (w = 0; w < 4; ++w) for (b = 0; b < 32; ++b) {
      if (jump[w] & (1u << b)) { acc[0] ^= s[0]; acc[1] ^= s[1]; acc[2] ^= s[2]; acc[3] ^= s[3]; }
      xb_rng_step(&s[0], &s[1], &s[2], &s[3]);
    }
    for (w = 0; w < 4; ++w) state[w * 16 + lane] = acc[w];
  }
}

LIBXSMM_API unsigned int* libxsmm_rng_create_extstate(unsigned int seed) {
  void* p = NULL;
  if (0 != posix_memalign(&p, 64, 64 * sizeof(unsigned int))) return NULL;
  xb_rng_seed_lanes(seed, (unsigned int*)p);
  return (unsigned int*)p;
}
LIBXSMM_API unsigned int libxsmm_rng_get_extstate_size(void) { return (unsigned int)(64 * sizeof(unsigned int)); }
LIBXSMM_API void libxsmm_rng_destroy_extstate(unsigned int* stateptr) { free(stateptr); }

/* f32 -> bf8 with a random byte added below the kept bits (src/libxsmm_lpflt_quant.c:303-368): element j draws from lane
 * (start_seed_idx + j % 16) % 16 of the caller's state (one xoshiro128++ step); f16-subnormal magnitudes round to nearest even, Inf/NaN pass */
LIBXSMM_API void libxsmm_stochastic_convert_fp32_bf8(const float* in, libxsmm_bfloat8* out, unsigned int len, void* rng_state, unsigned int start_seed_idx) {
  unsigned int* st = (unsigned int*)rng_state;
  unsigned int i;
  for (i = 0; i < len; ++i) {
    const unsigned int lane = (start_seed_idx + (i % 16)) % 16;
    const unsigned int sum = st[lane] + st[48 + lane], draw = ((sum << 7) | (sum >> 25)) + st[lane];
    unsigned int h = libxsmm_convert_f32_to_f16(in[i]);
    xb_rng_step(&st[lane], &st[16 + lane], &st[32 + lane], &st[48 + lane]);
    if ((h & 0x7c00u) == 0x7c00u) { if (h & 0x03ffu) h |= 0x0200u; }
    else if ((h & 0x7c00u) == 0u) h = (h + 0x7fu + ((h >> 8) & 1u)) & 0xffffu;
    else h = (h + (draw >> 24)) & 0xffffu;
    out[i] = (libxsmm_bfloat8)(h >> 8);
  }
}

LIBXSMM_API void libxsmm_rng_set_seed(unsigned int seed) {
  xb_rng_seed_lanes(seed, &g_rng[0][0]);
  srand(seed);                          /* the scalar draws below come from the C library, like the reference's */
  g_rng_seeded = 1;
}

LIBXSMM_API void libxsmm_rng_f32_seq(float* rngs, libxsmm_blasint count) {
  libxsmm_blasint i;
  if (!g_rng_seeded) libxsmm_rng_set_seed(0);
  for (i = 0; i < count; ++i) {
    const int lane = (int)(i & 15);
    union { unsigned int u; float f; } v;
    v.u = 0x3f800000u | ((g_rng[0][lane] + g_rng[3][lane]) >> 9);      /* [1, 2) from the top 23 bits */
    xb_rng_step(&g_rng[0][lane], &g_rng[1][lane], &g_rng[2][lane], &g_rng[3][lane]);
    rngs[i] = v.f - 1.0f;
  }
}

/* scalar draws come from the C library's rand(), like the reference as it builds (src/libxsmm_utils.c:20-83 picks
 * drand48 only under feature macros its own headers do not set): same seed, same sequence as the reference's drivers see */
LIBXSMM_API unsigned int libxsmm_rng_u32(unsigned int n) {
  const unsigned int rmax = (unsigned int)RAND_MAX + 1u;          /* rejection sampling removes the modulo bias */
  unsigned int r, nmax, q;
  if (n <= 1) return 0;
  nmax = (n < rmax) ? n : rmax; q = (rmax / nmax) * nmax;
  do { r = (unsigned int)rand(); } while (q <= r);
  if (n <= nmax) return r % nmax;
  return (unsigned int)(((double)n / nmax) * r + 0.5);
}

LIBXSMM_API void libxsmm_rng_seq(void* data, size_t nbytes) {
  unsigned char* dst = (unsigned char*)data;
  size_t done = 0;
  while (done < nbytes) {
    const unsigned int r = (unsigned int)rand();
    const size_t chunk = (nbytes - done < 4) ? (nbytes - done) : 4;
    memcpy(dst + done, &r, chunk); done += chunk;
  }
}

LIBXSMM_API double libxsmm_rng_f64(void) { return (1.0 / (RAND_MAX)) * (double)rand(); }

/* ---- low-precision array conversions ---------------------------------------------------------------------------- */
/* both flush f32 denormals to signed zero and quiet NaNs like the RNE converter (reference src/libxsmm_math.c:646-681) */
static unsigned int xb_bf16_prepare(float f, unsigned int round_add) {
  unsigned int u = xb_f32_bits(f);
  if ((u & 0x7f800000u) == 0u) u &= 0x80000000u;
  if ((u & 0x7f800000u) == 0x7f800000u) { if ((u & 0x007fffffu) != 0u) u |= 0x00400000u; }
  else u += round_add;
  return u;
}
LIBXSMM_API void libxsmm_truncate_convert_f32_bf16(const float* in, libxsmm_bfloat16* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = (libxsmm_bfloat16)(xb_bf16_prepare(in[i], 0u) >> 16);
}
LIBXSMM_API void libxsmm_rnaz_convert_fp32_bf16(const float* in, libxsmm_bfloat16* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = (libxsmm_bfloat16)(xb_bf16_prepare(in[i], 0x00008000u) >> 16);   /* ties away from zero */
}
LIBXSMM_API void libxsmm_rne_convert_fp32_bf16(const float* in, libxsmm_bfloat16* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = libxsmm_convert_f32_to_bf16_rne(in[i]);
}
LIBXSMM_API void libxsmm_convert_bf16_f32(const libxsmm_bfloat16* in, float* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = libxsmm_convert_bf16_to_f32(in[i]);
}
LIBXSMM_API void libxsmm_rne_convert_fp32_f16(const float* in, libxsmm_float16* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = libxsmm_convert_f32_to_f16(in[i]);
}
LIBXSMM_API void libxsmm_convert_f16_f32(const libxsmm_float16* in, float* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = libxsmm_convert_f16_to_f32(in[i]);
}

LIBXSMM_API void libxsmm_rne_convert_fp32_bf8(const float* in, libxsmm_bfloat8* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = xb_f32_to_bf8(in[i]);
}
LIBXSMM_API void libxsmm_convert_bf8_f32(const libxsmm_bfloat8* in, float* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = libxsmm_convert_f16_to_f32((libxsmm_float16)((unsigned short)in[i] << 8));
}
LIBXSMM_API void libxsmm_rne_convert_fp32_hf8(const float* in, libxsmm_hfloat8* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = xb_f32_to_hf8(in[i]);
}
LIBXSMM_API void libxsmm_convert_hf8_f32(const libxsmm_hfloat8* in, float* out, size_t length) {
  size_t i; for (i = 0; i < length; ++i) out[i] = xb_hf8_to_f32(in[i]);
}

/* ---- target queries ------------------------------------------------------------------------------------------------ */
LIBXSMM_API int libxsmm_cpuid(libxsmm_cpuid_info* info) {
  if (info != NULL) { memset(info, 0, sizeof(*info)); strncpy(info->model, "NVIDIA H100 (sm_90a)", sizeof(info->model) - 1); }
  return LIBXSMM_B200_SM90A;
}
LIBXSMM_API int libxsmm_cpuid_dot_pack_factor(libxsmm_datatype datatype) {
  const int ts = (int)libxsmm_typesize(datatype);
  return (ts == 2) ? 2 : ((ts == 1) ? 4 : 1);
}
LIBXSMM_API int libxsmm_cpuid_vlen32(int id) { (void)id; return 16; }   /* the reference's 512-bit lane count: dropout RNG consumption is defined on it */

LIBXSMM_API const char* libxsmm_stristr(const char a[], const char b[]) {
  const char* p;
  size_t nb;
  if (a == NULL || b == NULL) return NULL;
  nb = strlen(b);
  for (p = a; *p != 0; ++p) {
    size_t i = 0;
    while (i < nb && p[i] != 0 && tolower((unsigned char)p[i]) == tolower((unsigned char)b[i])) ++i;
    if (i == nb) return p;
  }
  return (nb == 0) ? a : NULL;
}
