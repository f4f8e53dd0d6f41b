/* libxsmm_b200 -- host runtime in plain C: library state, the handle registry, the dense
 * GEMM/BRGEMM dispatch and invocation path, batch entry points and kernel introspection.
 *
 * Role in the reference: src/libxsmm_main.c (registry + libxsmm_build + dispatch, :2132-3446) and
 * src/libxsmm_generator.c (descriptor construction, :143-321). There is no code generation here:
 * a handle is one of XB_NTHUNKS pre-compiled trampolines (host_thunks.c) whose index selects a slot
 * holding the normalised descriptor; calling it launches a pre-compiled sm_90a kernel.
 * No CUDA header is included: all device work goes through xb_rt_* and xb_*_launch (C ABI).
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"
#include "xb_device.cuh"

/* ---- public state words ------------------------------------------------------------------------ */
__attribute__((visibility("default"))) unsigned int libxsmm_ninit = 0;
__attribute__((visibility("default"))) int libxsmm_target_archid = 1000;  /* the backend's arch id: an ABI value drivers compare with the LIBXSMM_X86_* ids */
__attribute__((visibility("default"))) int libxsmm_verbosity = 0;

static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;
static xb_slot g_slots[XB_NTHUNKS];
static int g_nregistered = 0;
static int g_force_simt = 0;

/* registry: open addressing over slot indices, keyed by (kind, descriptor bytes) */
#define XB_REG_CAP 16384
static int g_reg[XB_REG_CAP];      /* 0: empty, else slot+1 */
static size_t g_reg_size = 0;

static unsigned int xb_hash(const void* data, size_t n, unsigned int seed) {
  const unsigned char* p = (const unsigned char*)data;
  unsigned int h = 2166136261u ^ seed;
  size_t i;
  for (i = 0; i < n; ++i) { h ^= p[i]; h *= 16777619u; }
  return h;
}

static const void* xb_key_of(const xb_slot* s, size_t* size) {
  switch (s->kind) {
    case XB_KIND_GEMM: case XB_KIND_GEMM_EXT: case XB_KIND_TILECFG: *size = sizeof(xb_gemm_desc); return &s->u.gemm;
    case XB_KIND_MELTW: *size = sizeof(xb_meltw_desc); return &s->u.meltw;
    default: *size = 0; return NULL;
  }
}

/* finds or inserts a registered slot for (kind,key); returns slot index or -1 (registry full) */
static int xb_registry_get(int kind, const void* key, size_t key_size, unsigned int nflops) {
  unsigned int h = xb_hash(key, key_size, (unsigned int)kind) & (XB_REG_CAP - 1);
  int result = -1, probes;
  pthread_mutex_lock(&g_lock);
  for (probes = 0; probes < XB_REG_CAP; ++probes, h = (h + 1) & (XB_REG_CAP - 1)) {
    if (g_reg[h] == 0) break;
    else {
      const xb_slot* s = &g_slots[g_reg[h] - 1];
      size_t ks; const void* k = xb_key_of(s, &ks);
      if (s->kind == kind && ks == key_size && 0 == memcmp(k, key, key_size)) { result = g_reg[h] - 1; break; }
    }
  }
  if (result < 0 && probes < XB_REG_CAP && g_reg_size < (XB_REG_CAP / 2)) {
    int i;
    for (i = 0; i < XB_NTHUNKS; ++i) if (g_slots[i].kind == XB_KIND_FREE) break;
    if (i < XB_NTHUNKS) {
      xb_slot* s = &g_slots[i];
      memset(s, 0, sizeof(*s));
      s->kind = kind; s->registered = 1; s->nflops = nflops;
      memcpy(&s->u, key, key_size);
      g_reg[h] = i + 1; ++g_reg_size; ++g_nregistered;
      result = i;
    }
  }
  pthread_mutex_unlock(&g_lock);
  return result;
}

/* caller-owned slot (create_* kernels); -1 if the pool is exhausted */
static int xb_slot_alloc(int kind, unsigned int nflops) {
  int i, result = -1;
  pthread_mutex_lock(&g_lock);
  for (i = XB_NTHUNKS - 1; i >= 0; --i) if (g_slots[i].kind == XB_KIND_FREE) break;
  if (i >= 0) {
    memset(&g_slots[i], 0, sizeof(xb_slot));
    g_slots[i].kind = kind; g_slots[i].registered = 0; g_slots[i].nflops = nflops;
    result = i;
  }
  pthread_mutex_unlock(&g_lock);
  return result;
}

int xb_host_slot_alloc(int kind, unsigned int nflops) { return xb_slot_alloc(kind, nflops); }
int xb_host_registry_get(int kind, const void* key, size_t key_size, unsigned int nflops) { return xb_registry_get(kind, key, key_size, nflops); }
xb_slot* xb_host_slot(int i) { return (i >= 0 && i < XB_NTHUNKS) ? &g_slots[i] : NULL; }

static void xb_sparse_release(xb_sparse_desc* sp) {
  if (sp->d_ptr) xb_rt_device_free(sp->d_ptr);
  if (sp->d_idx) xb_rt_device_free(sp->d_idx);
  if (sp->d_val) xb_rt_device_free(sp->d_val);
  if (sp->work) xb_bcsc_state_free(sp->work);
  sp->d_ptr = NULL; sp->d_idx = NULL; sp->d_val = NULL; sp->work = NULL;
}

/* ---- lifetime ---------------------------------------------------------------------------------- */
extern void xb_thunks_init(void);

__attribute__((constructor)) static void xb_ctor(void) { libxsmm_init(); }

LIBXSMM_API void libxsmm_init(void) {
  pthread_mutex_lock(&g_lock);
  if (libxsmm_ninit < 2) {
    const char* env = getenv("LIBXSMM_VERBOSE");
    if (env != NULL && *env != 0) libxsmm_verbosity = atoi(env);
    env = getenv("LIBXSMM_B200_FORCE_SIMT");
    if (env != NULL && *env != 0) g_force_simt = atoi(env);
    xb_thunks_init();
    libxsmm_ninit = 2;
  }
  pthread_mutex_unlock(&g_lock);
}

LIBXSMM_API void libxsmm_finalize(void) {
  int i;
  pthread_mutex_lock(&g_lock);
  for (i = 0; i < XB_NTHUNKS; ++i) {
    xb_slot* s = &g_slots[i];
    if (s->kind != XB_KIND_FREE && s->registered) { memset(s, 0, sizeof(*s)); }
  }
  memset(g_reg, 0, sizeof(g_reg));
  g_reg_size = 0; g_nregistered = 0;
  if (libxsmm_verbosity != 0) {
    fprintf(stderr, "LIBXSMM-B200: %llu kernel launches, target %s\n", xb_rt_launch_count(), "sm_90a");
  }
  libxsmm_ninit = 0;
  pthread_mutex_unlock(&g_lock);
}

LIBXSMM_API int libxsmm_get_target_archid(void) { return libxsmm_target_archid; }
LIBXSMM_API void libxsmm_set_target_archid(int id) { (void)id; }
LIBXSMM_API const char* libxsmm_get_target_arch(void) { return "sm_90a"; }
LIBXSMM_API void libxsmm_set_target_arch(const char* arch) { (void)arch; }
LIBXSMM_API int libxsmm_get_verbosity(void) { return libxsmm_verbosity; }
LIBXSMM_API void libxsmm_set_verbosity(int level) { libxsmm_verbosity = level; }

static const struct { const char* name; unsigned char size; } g_types[] = {
#define XB_X(NAME, BYTES) { #NAME, BYTES },
  LIBXSMM_B200_DATATYPES(XB_X)
#undef XB_X
};

LIBXSMM_API unsigned char libxsmm_typesize(libxsmm_datatype datatype) {
  return ((int)datatype >= 0 && (int)datatype < LIBXSMM_DATATYPE_B200_COUNT) ? g_types[datatype].size : 0;
}

LIBXSMM_API const char* libxsmm_get_typename(libxsmm_datatype datatype) {
  static const char* const lower[] = { "f64", "f32", "bf16", "f16", "bf8", "hf8", "i64", "u64", "i32", "u32", "i16",
    "u16", "i8", "u8", "mxbf8", "mxhf8", "mxbf6", "mxhf6", "i4x2", "u4x2", "mxfp4x2", "nvfp4x2", "i2x4", "i1x8", "bf32",
    "implicit", "unsupported" };
  return ((int)datatype >= 0 && (int)datatype < LIBXSMM_DATATYPE_B200_COUNT) ? lower[datatype] : "void";
}

/* ---- conversions (host twins of the device helpers) -------------------------------------------- */
LIBXSMM_API float libxsmm_convert_bf16_to_f32(libxsmm_bfloat16 in) {
  /* the stand-alone converter flushes bf16 denormals (reference src/libxsmm_math.c:587-597) */
  if ((in & 0x7f80) == 0) in = (libxsmm_bfloat16)(in & 0x8000);
  return xb_bf16_to_f32(in);
}
LIBXSMM_API float libxsmm_convert_f16_to_f32(libxsmm_float16 in) { return xb_f16_to_f32(in); }
LIBXSMM_API libxsmm_bfloat16 libxsmm_convert_f32_to_bf16_rne(float in) { return xb_f32_to_bf16_rne(in); }
LIBXSMM_API libxsmm_float16 libxsmm_convert_f32_to_f16(float in) { return xb_f32_to_f16(in); }

/* ---- memory ------------------------------------------------------------------------------------ */
LIBXSMM_API void* libxsmm_aligned_malloc(size_t size, size_t alignment) {
  void* p = NULL;
  (void)alignment;                      /* CUDA allocations are at least 256-byte aligned */
  if (xb_rt_have_gpu()) p = xb_rt_managed_malloc(size);
  if (p == NULL) {                      /* no device (CPU-only host logic tests): plain aligned memory */
    if (0 != posix_memalign(&p, 256, size ? size : 1)) p = NULL;
  }
  return p;
}
LIBXSMM_API void* libxsmm_malloc(size_t size) { return libxsmm_aligned_malloc(size, 0); }
LIBXSMM_API void libxsmm_free(const void* memory) {
  if (memory == NULL) return;
  if (xb_rt_have_gpu() && xb_rt_ptr_kind(memory) == 2) xb_rt_managed_free((void*)(uintptr_t)memory);
  else free((void*)(uintptr_t)memory);
}

LIBXSMM_API int libxsmm_b200_device_count(void) { return xb_rt_device_count(); }
LIBXSMM_API int libxsmm_b200_set_device(int ordinal) { return xb_rt_set_device(ordinal); }
LIBXSMM_API void libxsmm_b200_set_stream(void* s) { xb_rt_set_stream(s); }
LIBXSMM_API void libxsmm_b200_set_blocking(int b) { xb_rt_set_blocking(b); }
LIBXSMM_API int libxsmm_b200_sync(void) { return xb_rt_sync(); }
LIBXSMM_API int libxsmm_b200_last_error(void) { return xb_rt_last_error(); }
LIBXSMM_API const char* libxsmm_b200_last_error_string(void) { return xb_rt_last_error_string(); }
LIBXSMM_API unsigned long long libxsmm_b200_launch_count(void) { return xb_rt_launch_count(); }
LIBXSMM_API void libxsmm_b200_set_force_simt(int on) { g_force_simt = on; }
LIBXSMM_API void* libxsmm_b200_device_malloc(size_t size) { return xb_rt_device_malloc(size); }
LIBXSMM_API void libxsmm_b200_device_free(void* p) { xb_rt_device_free(p); }
LIBXSMM_API void* libxsmm_b200_host_malloc(size_t size) { return xb_rt_host_malloc(size); }
LIBXSMM_API void libxsmm_b200_host_free(void* p) { xb_rt_host_free(p); }
LIBXSMM_API int libxsmm_b200_memcpy(void* dst, const void* src, size_t size) { return xb_rt_memcpy(dst, src, size); }

/* ---- shape/config constructors ----------------------------------------------------------------- */
LIBXSMM_API libxsmm_gemm_shape libxsmm_create_gemm_shape(libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint k,
  libxsmm_blasint lda, libxsmm_blasint ldb, libxsmm_blasint ldc,
  libxsmm_datatype a_in_type, libxsmm_datatype b_in_type, libxsmm_datatype out_type, libxsmm_datatype comp_type)
{
  libxsmm_gemm_shape s;
  memset(&s, 0, sizeof(s));
  s.m = m; s.n = n; s.k = k; s.lda = lda; s.ldb = ldb; s.ldc = ldc;
  s.a_in_type = a_in_type; s.b_in_type = b_in_type; s.out_type = out_type; s.comp_type = comp_type;
  return s;
}

LIBXSMM_API libxsmm_gemm_batch_reduce_config libxsmm_create_gemm_batch_reduce_config(
  libxsmm_gemm_batch_reduce_type br_type, libxsmm_blasint br_stride_a_hint, libxsmm_blasint br_stride_b_hint,
  unsigned char br_unroll_hint)
{
  libxsmm_gemm_batch_reduce_config c;
  memset(&c, 0, sizeof(c));
  c.br_type = br_type; c.br_stride_a_hint = br_stride_a_hint; c.br_stride_b_hint = br_stride_b_hint;
  c.br_unroll_hint = br_unroll_hint;
  return c;
}

LIBXSMM_API libxsmm_gemm_ext_unary_argops libxsmm_create_gemm_ext_unary_argops(
  libxsmm_blasint ldap, libxsmm_meltw_unary_type ap_unary_type, libxsmm_bitfield ap_unary_flags, libxsmm_blasint store_ap,
  libxsmm_blasint ldbp, libxsmm_meltw_unary_type bp_unary_type, libxsmm_bitfield bp_unary_flags, libxsmm_blasint store_bp,
  libxsmm_blasint ldcp, libxsmm_meltw_unary_type cp_unary_type, libxsmm_bitfield cp_unary_flags, libxsmm_blasint store_cp)
{
  libxsmm_gemm_ext_unary_argops r;
  memset(&r, 0, sizeof(r));
  r.ldap = ldap; r.ap_unary_type = ap_unary_type; r.ap_unary_flags = ap_unary_flags; r.store_ap = store_ap;
  r.ldbp = ldbp; r.bp_unary_type = bp_unary_type; r.bp_unary_flags = bp_unary_flags; r.store_bp = store_bp;
  r.ldcp = ldcp; r.cp_unary_type = cp_unary_type; r.cp_unary_flags = cp_unary_flags; r.store_cp = store_cp;
  return r;
}

LIBXSMM_API libxsmm_gemm_ext_binary_postops libxsmm_create_gemm_ext_binary_postops(
  libxsmm_blasint ldd, libxsmm_datatype d_in_type, libxsmm_meltw_binary_type d_binary_type, libxsmm_bitfield d_binary_flags)
{
  libxsmm_gemm_ext_binary_postops r;
  memset(&r, 0, sizeof(r));
  r.ldd = ldd; r.d_in_type = d_in_type; r.d_binary_type = d_binary_type; r.d_binary_flags = d_binary_flags;
  return r;
}

/* ---- dense GEMM dispatch ------------------------------------------------------------------------ */
static int xb_tilecfg_inconsistent(unsigned int flags) {
  /* exactly one of NO_RESET/NO_SETUP set => tile-config handle, not a GEMM (reference
   * src/libxsmm_generator.c:154-157): the GEMM dispatchers answer NULL */
  const int nr = (flags & LIBXSMM_GEMM_FLAG_NO_RESET_TILECONFIG) != 0;
  const int ns = (flags & LIBXSMM_GEMM_FLAG_NO_SETUP_TILECONFIG) != 0;
  return nr != ns;
}

/* A's layout (gemm_simt.cu gives the formulas): the VNNI factor its k is packed by (1: not packed) and, in *trans, whether TRANS_A
 * is honoured. F64 / F32 / BF32 A are read flat whatever VNNI_A says; an int8 A next to an f32 C is always VNNI4; an 8-bit float A
 * is VNNI4, or VNNI2 next to a bf16 B. The narrow forms (MX fp8, dequantising, low-bit) read A in layouts of their own. */
static int xb_layout_a(const xb_gemm_desc* d, int* trans) {
  const int ta = d->ta, is8 = (ta == LIBXSMM_DATATYPE_I8 || ta == LIBXSMM_DATATYPE_U8), is_f8 = (ta == LIBXSMM_DATATYPE_BF8 || ta == LIBXSMM_DATATYPE_HF8);
  const int flat = (ta == LIBXSMM_DATATYPE_F64 || ta == LIBXSMM_DATATYPE_F32 || ta == LIBXSMM_DATATYPE_BF32);
  *trans = (d->flags & LIBXSMM_GEMM_FLAG_TRANS_A) != 0 && (flat || ta == LIBXSMM_DATATYPE_BF16 || is_f8);
  if ((d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0 ? flat : !(is8 && d->tc == LIBXSMM_DATATYPE_F32)) return 1;
  return (is8 || (is_f8 && d->tb != LIBXSMM_DATATYPE_BF16)) ? 4 : 2;
}

/* B's layout: the VNNI factor of its transposed, packed form (1: not packed) and, in *trans, whether TRANS_B is honoured. A bf16
 * B under TRANS_B and VNNI_B is VNNI2-T, an MX fp8 B VNNI4-T. */
static int xb_layout_b(const xb_gemm_desc* d, int* trans) {
  const int tb = d->tb, mx = (tb == LIBXSMM_DATATYPE_MXBF8 || tb == LIBXSMM_DATATYPE_MXHF8);
  *trans = (d->flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0 && (mx || tb == LIBXSMM_DATATYPE_F64 || tb == LIBXSMM_DATATYPE_F32 || tb == LIBXSMM_DATATYPE_BF32
                                                           || tb == LIBXSMM_DATATYPE_BF16 || tb == LIBXSMM_DATATYPE_F16 || tb == LIBXSMM_DATATYPE_BF8 || tb == LIBXSMM_DATATYPE_HF8);
  if (mx) return 4;
  return (*trans && (d->flags & LIBXSMM_GEMM_FLAG_VNNI_B) != 0 && tb == LIBXSMM_DATATYPE_BF16) ? 2 : 1;
}

/* The exact-order path that serves a GEMM descriptor, or XB_PATH_NONE: the one rule for which type tuples, flags, leading dimensions,
 * divisibilities, batch-reduce modes and fusions dispatch. Line numbers cite the reference's src/generator_gemm_reference_impl.c.
 * The narrow A forms (MX fp8, dequantising, low-bit) exist for the plain ABI only and decline every flag the reference would ignore
 * rather than obey, so that no caller gets a layout other than the one asked for. */
int xb_gemm_path(const xb_gemm_desc* d) {
  const unsigned int f = d->flags;
  const int ta = d->ta, tb = d->tb, tc = d->tc, comp = d->tcomp;
  const int ext = (f & LIBXSMM_GEMM_FLAG_USE_XGEMM_EXT_ABI) != 0, vnni_a = (f & LIBXSMM_GEMM_FLAG_VNNI_A) != 0;
  const int a8 = (ta == LIBXSMM_DATATYPE_I8 || ta == LIBXSMM_DATATYPE_U8), b8 = (tb == LIBXSMM_DATATYPE_I8 || tb == LIBXSMM_DATATYPE_U8);
  const int a4 = (ta == LIBXSMM_DATATYPE_I4X2 || ta == LIBXSMM_DATATYPE_U4X2), b16 = (tb == LIBXSMM_DATATYPE_BF16 || tb == LIBXSMM_DATATYPE_F16);
  const int a_f8 = (ta == LIBXSMM_DATATYPE_BF8 || ta == LIBXSMM_DATATYPE_HF8), a_mx = (ta == LIBXSMM_DATATYPE_MXBF8 || ta == LIBXSMM_DATATYPE_MXHF8);
  int trans_a, trans_b, path = XB_PATH_NONE;
  const int va = xb_layout_a(d, &trans_a);
  xb_layout_b(d, &trans_b);
  if (d->lda < (trans_a ? d->k : d->m) || d->ldb < (trans_b ? d->n : d->k)) return XB_PATH_NONE;
  if (a_mx || tb == LIBXSMM_DATATYPE_MXBF8 || tb == LIBXSMM_DATATYPE_MXHF8 || tc == LIBXSMM_DATATYPE_MXBF8 || tc == LIBXSMM_DATATYPE_MXHF8) {
    /* MXBF8 x MXBF8 and MXHF8 x MXHF8 with E8M0 block scales (:2620-2679); every other MX tuple matches no branch. The reference
     * prints an error and leaves C without VNNI_A, VNNI_B and TRANS_B (:2632-2635). */
    const unsigned int need = LIBXSMM_GEMM_FLAG_VNNI_A | LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_TRANS_B;
    const int mx_c = (tc == LIBXSMM_DATATYPE_MXBF8);
    if (ext || !a_mx || tb != ta || comp != LIBXSMM_DATATYPE_F32 || !(tc == LIBXSMM_DATATYPE_F32 || (mx_c && ta == LIBXSMM_DATATYPE_MXBF8))) return XB_PATH_NONE;
    if ((f & (need | LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_VNNI_C | LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK)) != need || (d->k % 32) != 0) return XB_PATH_NONE;
    /* block r is read at r*lda*k and r*ldb*k whatever the batch-reduce type says (:2646-2655): stride mode only where the hints agree;
     * address and offset mode would read the pointer / offset arrays as data, which defines no result */
    if (d->br_type == 1 || d->br_type == 2) return XB_PATH_NONE;
    if (d->br_type == 3 && (d->br_stride_a != (long long)d->lda * d->k || d->br_stride_b != (long long)d->ldb * d->k)) return XB_PATH_NONE;
    /* MXBF8 C: the reference accumulates into an uninitialised image unless beta = 0, and quantises whole 32-row blocks (:757-) */
    if (mx_c && ((f & LIBXSMM_GEMM_FLAG_BETA_0) == 0 || (d->m % 32) != 0 || (d->ldc % 32) != 0)) return XB_PATH_NONE;
    return P_MX8;
  }
  if (((a8 || a4) && b16) || (ta == LIBXSMM_DATATYPE_BF8 && tb == LIBXSMM_DATATYPE_F16)) {
    /* dequantising A (xb_dq_form, :1684-2024), and its unsigned / mis-typed neighbours. No branch reads A transposed or B / C
     * VNNI-packed; bitmap A is the sparse branch (:857-948); INTLV_A_FORMAT makes int4 the int8-B form (:472-480). */
    const int form = xb_dq_form(d);
    if (ext || form == XB_DQ_NONE || (f & (LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_VNNI_C
                                           | LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT)) != 0) return XB_PATH_NONE;
    if (form == XB_DQ_I8_BF16 && trans_b) return XB_PATH_NONE;                                   /* B is read [n][ldb] whatever the flag says (:1709) */
    if ((form == XB_DQ_I8_BF16 || form == XB_DQ_I8_F16) && vnni_a) return XB_PATH_NONE;          /* A is read flat (l_k_block = 1, :1691, :1891, :1963) */
    if (form == XB_DQ_I4_F16 && !vnni_a) return XB_PATH_NONE;                                    /* int4 x f16 is the VNNI_A form only (:472) */
    if ((form == XB_DQ_I4_F16 || (form == XB_DQ_BF8_F16 && vnni_a)) && (d->k % 2) != 0) return XB_PATH_NONE;   /* k in pairs: an odd k would drop the last */
    return P_DQ;
  }
  if (ta == LIBXSMM_DATATYPE_I2X4 || ta == LIBXSMM_DATATYPE_I1X8 || (ta == LIBXSMM_DATATYPE_MXFP4X2 && b8)) {
    /* low-bit A (xb_lowbit_form, :1009-1272, set-up :457-490, :560-620), and its mis-typed neighbours. Every branch reads A in its
     * packed layout, B as [n][ldb] and C flat; bitmap A is the sparse branch (:857-948). */
    const int form = xb_lowbit_form(d);
    const unsigned int packed = f & (LIBXSMM_GEMM_FLAG_VNNI_A | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT);
    if (ext || form == XB_LB_NONE || (f & (LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B | LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_VNNI_C
                                           | LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK)) != 0) return XB_PATH_NONE;
    switch (form) {
      case XB_LB_I2:   /* :482; rows past 4*(m/4) and k past 4*(k/4) would be left out */
        return (packed == (LIBXSMM_GEMM_FLAG_VNNI_A | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT) && (d->m % 4) == 0 && (d->k % 4) == 0) ? P_LOWBIT : XB_PATH_NONE;
      case XB_LB_I1:   /* :486 ignores INTLV_A_FORMAT; rows come in pairs (:1204) and k in fours (:1211) */
        return (packed == LIBXSMM_GEMM_FLAG_VNNI_A && (d->m % 2) == 0 && (d->k % 4) == 0 && (d->lda % 2) == 0) ? P_LOWBIT : XB_PATH_NONE;
      default:         /* MXFP4: :467, 32-k scale blocks */
        return (packed == (LIBXSMM_GEMM_FLAG_VNNI_A | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT) && (d->k % 32) == 0) ? P_LOWBIT : XB_PATH_NONE;
    }
  }
  /* every other A: the layout of xb_layout_a / xb_layout_b, a 16-bit C in column pairs under VNNI_C */
  if ((a_f8 && vnni_a && trans_a) || (d->k % va) != 0) return XB_PATH_NONE;
  if ((f & LIBXSMM_GEMM_FLAG_VNNI_C) != 0 && ((d->n % 2) != 0 || libxsmm_typesize((libxsmm_datatype)tc) != 2)) return XB_PATH_NONE;
  if ((f & LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK) != 0) {   /* bitmap-compressed A (:857-948): float operands, no batch reduce */
    const int fa = (ta == LIBXSMM_DATATYPE_F32 || ta == LIBXSMM_DATATYPE_BF16 || ta == LIBXSMM_DATATYPE_F16);
    const int fb = (tb == LIBXSMM_DATATYPE_F32 || tb == LIBXSMM_DATATYPE_BF16 || tb == LIBXSMM_DATATYPE_F16);
    const int fc = (tc == LIBXSMM_DATATYPE_F32 || tc == LIBXSMM_DATATYPE_BF16 || tc == LIBXSMM_DATATYPE_F16);
    const int kb = (ta == LIBXSMM_DATATYPE_F32 || tb == LIBXSMM_DATATYPE_F32) ? 1 : 2;
    if (fa && fb && fc && d->br_type == 0 && (d->k % kb) == 0) path = P_BITMAP;
  } else if (a4) {   /* 4-bit A with zero points x 8-bit B -> I32 (:1273-1321) */
    const unsigned int need = LIBXSMM_GEMM_FLAG_VNNI_A | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT;
    if ((f & need) == need && b8 && tc == LIBXSMM_DATATYPE_I32 && comp == LIBXSMM_DATATYPE_I32 && (d->k % 8) == 0 && (d->br_type == 0 || d->br_type == 3)) path = P_I4_I32;
  } else {
    const int f16comp = (comp == LIBXSMM_DATATYPE_F16 || comp == LIBXSMM_DATATYPE_F32 || comp == LIBXSMM_DATATYPE_IMPLICIT);
    if (ta == LIBXSMM_DATATYPE_F64 && tb == ta && tc == ta && comp == ta) path = P_F64;
    else if ((ta == LIBXSMM_DATATYPE_F32 || ta == LIBXSMM_DATATYPE_BF32) && (tb == LIBXSMM_DATATYPE_F32 || tb == LIBXSMM_DATATYPE_BF32)
             && tc == LIBXSMM_DATATYPE_F32 && comp == LIBXSMM_DATATYPE_F32) path = P_F32;
    else if (ta == LIBXSMM_DATATYPE_I16 && tb == ta && tc == LIBXSMM_DATATYPE_I32 && comp == LIBXSMM_DATATYPE_I32) path = P_I16;
    else if (a8 && b8 && tc == LIBXSMM_DATATYPE_I32 && comp == LIBXSMM_DATATYPE_I32) path = P_I8_I32;
    else if (a8 && b8 && tc == LIBXSMM_DATATYPE_F32 && comp == LIBXSMM_DATATYPE_I32) path = P_I8_F32;
    else if (ta == LIBXSMM_DATATYPE_F16 && tb == ta && tc == LIBXSMM_DATATYPE_F16 && f16comp) path = P_F16_F16;
    else if (ta == LIBXSMM_DATATYPE_F16 && tb == ta && tc == LIBXSMM_DATATYPE_F32 && f16comp) path = P_F16_F32;
    else if (ta == LIBXSMM_DATATYPE_BF16 && tb == ta && tc == LIBXSMM_DATATYPE_F32 && comp == LIBXSMM_DATATYPE_F32) path = P_BF16_F32;
    else if (ta == LIBXSMM_DATATYPE_BF16 && tb == ta && tc == LIBXSMM_DATATYPE_BF16 && comp == LIBXSMM_DATATYPE_F32) path = P_BF16_BF16;
    /* 8-bit float A (:2171-2366 with a bf16 B, :2420-2630 with B and C of A's type or f32): f32 accumulate, one rounding */
    else if (a_f8 && comp == LIBXSMM_DATATYPE_F32 && (f & (LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_VNNI_C)) == 0
             && ((tb == ta && (tc == LIBXSMM_DATATYPE_F32 || tc == ta)) || (tb == LIBXSMM_DATATYPE_BF16 && (tc == LIBXSMM_DATATYPE_F32 || tc == LIBXSMM_DATATYPE_BF16)))) path = P_FP8;
  }
  if (d->fuse_colbias != 0 || d->cp_op != 0) {   /* fused form: float C only (the reference's f32 image of C) */
    return (path == P_F32 || path == P_I8_F32 || path == P_F16_F16 || path == P_F16_F32 || path == P_BF16_F32 || path == P_BF16_BF16) ? path : XB_PATH_NONE;
  }
  return path;
}

static int xb_make_gemm_desc(xb_gemm_desc* d, const libxsmm_gemm_shape* shape, unsigned int flags, unsigned int prefetch,
                             const libxsmm_gemm_batch_reduce_config* br, int ext)
{
  memset(d, 0, sizeof(*d));
  if (shape->m <= 0 || shape->n <= 0 || shape->k <= 0) return 0;
  if (shape->lda <= 0 || shape->ldb <= 0 || shape->ldc < shape->m) return 0;
  d->m = shape->m; d->n = shape->n; d->k = shape->k; d->lda = shape->lda; d->ldb = shape->ldb; d->ldc = shape->ldc;
  d->ta = (int)shape->a_in_type; d->tb = (int)shape->b_in_type; d->tc = (int)shape->out_type; d->tcomp = (int)shape->comp_type;
  /* the ABI flag says which dispatcher made the handle, whatever the caller passed */
  d->flags = (flags & ~(unsigned int)(LIBXSMM_GEMM_FLAG_USE_XGEMM_ABI | LIBXSMM_GEMM_FLAG_USE_XGEMM_EXT_ABI))
           | (ext ? LIBXSMM_GEMM_FLAG_USE_XGEMM_EXT_ABI : LIBXSMM_GEMM_FLAG_USE_XGEMM_ABI);
  d->prefetch = (int)prefetch;
  if (br != NULL) {
    switch ((int)br->br_type) {
      case LIBXSMM_GEMM_BATCH_REDUCE_ADDRESS: d->br_type = 1; d->flags |= LIBXSMM_GEMM_FLAG_BATCH_REDUCE_ADDRESS; break;
      case LIBXSMM_GEMM_BATCH_REDUCE_OFFSET: d->br_type = 2; d->flags |= LIBXSMM_GEMM_FLAG_BATCH_REDUCE_OFFSET; break;
      case LIBXSMM_GEMM_BATCH_REDUCE_STRIDE: d->br_type = 3; d->flags |= LIBXSMM_GEMM_FLAG_BATCH_REDUCE_STRIDE;
        d->br_stride_a = br->br_stride_a_hint; d->br_stride_b = br->br_stride_b_hint; break;
      default: d->br_type = 0;
    }
    if (d->br_type != 0) d->br_unroll = (br->br_unroll_hint > 0 && br->br_unroll_hint < 255) ? br->br_unroll_hint : 0;
  }
  d->path = xb_gemm_path(d);
  if (d->path == XB_PATH_NONE) return 0;
  d->backend = (!g_force_simt && (xb_gemm_tc_supported(d) || xb_gemm_ts_supported(d))) ? LIBXSMM_B200_BACKEND_TCGEN05 : LIBXSMM_B200_BACKEND_SIMT;
  return 1;
}

static libxsmm_gemmfunction xb_dispatch_gemm_common(const libxsmm_gemm_shape* shape, unsigned int flags, unsigned int prefetch,
                                                    const libxsmm_gemm_batch_reduce_config* br)
{
  xb_gemm_desc d;
  int slot;
  LIBXSMM_INIT
  if (xb_tilecfg_inconsistent(flags)) return NULL;
  if (!xb_make_gemm_desc(&d, shape, flags, prefetch, br, 0)) return NULL;
  slot = xb_registry_get(XB_KIND_GEMM, &d, sizeof(d), 2u * (unsigned int)d.m * (unsigned int)d.n * (unsigned int)d.k);
  return (slot < 0) ? NULL : (libxsmm_gemmfunction)xb_thunk(slot);
}

LIBXSMM_API libxsmm_gemmfunction libxsmm_dispatch_gemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags)
{
  return xb_dispatch_gemm_common(&gemm_shape, gemm_flags, prefetch_flags, NULL);
}

LIBXSMM_API libxsmm_gemmfunction libxsmm_dispatch_brgemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags,
  const libxsmm_gemm_batch_reduce_config brgemm_config)
{
  return xb_dispatch_gemm_common(&gemm_shape, gemm_flags, prefetch_flags, &brgemm_config);
}

LIBXSMM_API libxsmm_gemmfunction_ext libxsmm_dispatch_brgemm_ext(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags,
  const libxsmm_gemm_batch_reduce_config brgemm_config,
  const libxsmm_gemm_ext_unary_argops unary_argops, const libxsmm_gemm_ext_binary_postops binary_postops)
{
  xb_gemm_desc d;
  int slot;
  LIBXSMM_INIT
  if (xb_tilecfg_inconsistent(gemm_flags)) return NULL;
  /* the fusions the reference implements (generator_gemm_reference_impl.c:396-427): a column-broadcast bias added before the
   * product, ReLU (optionally recording a bitmask) or sigmoid applied to C; operand-side argops do not exist there either */
  if (unary_argops.ap_unary_type != LIBXSMM_MELTW_TYPE_UNARY_NONE || unary_argops.bp_unary_type != LIBXSMM_MELTW_TYPE_UNARY_NONE) return NULL;
  if (unary_argops.cp_unary_type != LIBXSMM_MELTW_TYPE_UNARY_NONE && unary_argops.cp_unary_type != LIBXSMM_MELTW_TYPE_UNARY_RELU
   && unary_argops.cp_unary_type != LIBXSMM_MELTW_TYPE_UNARY_SIGMOID) return NULL;
  if (binary_postops.d_binary_type != LIBXSMM_MELTW_TYPE_BINARY_NONE) {
    if (binary_postops.d_binary_type != LIBXSMM_MELTW_TYPE_BINARY_ADD) return NULL;
    if ((binary_postops.d_binary_flags & (LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_0 | LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_1)) == 0) return NULL;
  }
  if (!xb_make_gemm_desc(&d, &gemm_shape, gemm_flags, prefetch_flags, &brgemm_config, 1)) return NULL;
  if (unary_argops.cp_unary_type != LIBXSMM_MELTW_TYPE_UNARY_NONE || binary_postops.d_binary_type != LIBXSMM_MELTW_TYPE_BINARY_NONE) {
    d.fuse_colbias = (binary_postops.d_binary_type == LIBXSMM_MELTW_TYPE_BINARY_ADD); d.d_type = d.tc; d.ldd = binary_postops.ldd;
    d.cp_op = (int)unary_argops.cp_unary_type; d.cp_flags = (int)(unary_argops.cp_unary_flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT); d.ldcp = unary_argops.ldcp;
    d.path = xb_gemm_path(&d);
    if (d.path == XB_PATH_NONE) return NULL;             /* float C only */
    d.backend = LIBXSMM_B200_BACKEND_SIMT;               /* the fused epilogue lives in the exact-order kernel */
  }
  slot = xb_registry_get(XB_KIND_GEMM_EXT, &d, sizeof(d), 2u * (unsigned int)d.m * (unsigned int)d.n * (unsigned int)d.k);
  return (slot < 0) ? NULL : (libxsmm_gemmfunction_ext)xb_thunk(slot);
}

LIBXSMM_API libxsmm_tilecfgfunction libxsmm_dispatch_tilecfg_gemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags)
{
  xb_gemm_desc d;
  int slot;
  LIBXSMM_INIT
  if (!xb_tilecfg_inconsistent(gemm_flags)) return NULL;   /* reference src/libxsmm_main.c:3355-3387 */
  memset(&d, 0, sizeof(d));
  d.m = gemm_shape.m; d.n = gemm_shape.n; d.k = gemm_shape.k; d.lda = gemm_shape.lda; d.ldb = gemm_shape.ldb; d.ldc = gemm_shape.ldc;
  d.ta = (int)gemm_shape.a_in_type; d.tb = (int)gemm_shape.b_in_type; d.tc = (int)gemm_shape.out_type; d.tcomp = (int)gemm_shape.comp_type;
  d.flags = gemm_flags; d.backend = LIBXSMM_B200_BACKEND_NOOP;
  slot = xb_registry_get(XB_KIND_TILECFG, &d, sizeof(d), 0);
  return (slot < 0) ? NULL : (libxsmm_tilecfgfunction)xb_thunk(slot);
}

/* ---- invocation of a dense GEMM handle ---------------------------------------------------------- */
typedef struct xb_copyback { void* host; const void* dev; size_t bytes; } xb_copyback;

static size_t xb_extent_a(const xb_gemm_desc* d) {   /* elements touched in one A operand */
  int trans, v;
  switch (d->path) {
    case P_DQ:       /* bytes: int4 pairs [k/2][lda], bf8 VNNI2 [k/2][lda][2], else flat [k][lda] */
      if (xb_dq_form(d) == XB_DQ_I4_F16) return (size_t)(d->k / 2 - 1) * d->lda + (size_t)d->m;
      if ((d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0) return (size_t)(d->k / 2 - 1) * d->lda * 2 + (size_t)d->m * 2;
      return (size_t)(d->k - 1) * d->lda + d->m;
    case P_LOWBIT:   /* bytes: I2 [k/4][lda], I1 [k/4][lda/2], MXFP4 [k/8][lda][4] */
      if (xb_lowbit_form(d) == XB_LB_I2) return (size_t)(d->k / 4 - 1) * d->lda + (size_t)d->m;
      if (xb_lowbit_form(d) == XB_LB_I1) return (size_t)(d->k / 4 - 1) * (d->lda / 2) + (size_t)(d->m / 2);
      return (size_t)(d->k / 8 - 1) * d->lda * 4 + (size_t)d->m * 4;
    case P_I4_I32: return (size_t)(d->k / 8 - 1) * d->lda * 4 + (size_t)d->m * 4;   /* bytes: 8 k per 4 bytes */
    case P_MX8: return (size_t)(d->k / 4 - 1) * d->lda * 4 + (size_t)d->m * 4;      /* VNNI4 */
    default: break;
  }
  v = xb_layout_a(d, &trans);
  if (v > 1) return (size_t)(d->k / v - 1) * d->lda * v + (size_t)d->m * v;
  if (trans && (d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) == 0) return (size_t)(d->m - 1) * d->lda + d->k;
  return (size_t)(d->k - 1) * d->lda + d->m;
}

static size_t xb_extent_b(const xb_gemm_desc* d) {
  int trans;
  const int v = xb_layout_b(d, &trans);
  if (v > 1) return (size_t)(d->k / v - 1) * d->ldb * v + (size_t)d->n * v;   /* VNNI-T */
  if (trans) return (size_t)(d->k - 1) * d->ldb + d->n;
  return (size_t)(d->n - 1) * d->ldb + d->k;
}

/* MX block scales touched by one call of br blocks: [br][k/32][ld] bytes, up to the last row in use */
static size_t xb_extent_mx_scales(const xb_gemm_desc* d, unsigned long long br, int ld, int rows) {
  return (size_t)((br ? br : 1) * (unsigned long long)(d->k / 32) - 1) * (size_t)ld + (size_t)rows;
}

/* returns a device-usable pointer for `p`: itself if the device can read it, else a staged copy */
static const void* xb_stage_in(const void* p, size_t bytes, int* staged) {
  if (p == NULL || xb_rt_ptr_kind(p) != 0) return p;
  else {
    void* dptr = xb_rt_scratch(bytes);
    if (dptr == NULL) return NULL;
    xb_rt_upload(dptr, p, bytes);
    *staged = 1;
    return dptr;
  }
}

/* an address-mode array of br pointers to side data of `bytes` bytes each (MXFP4 block scales): a device array is used as given,
 * a host-readable one is copied with each pointer made device-usable */
static const void* xb_stage_ptr_array(const void* arr, unsigned long long br, size_t bytes, int* staged) {
  const size_t nbytes = (size_t)(br ? br : 1) * sizeof(void*);
  const void** h; void* dev; unsigned long long r;
  if (arr == NULL || xb_rt_ptr_kind(arr) == 1) return arr;
  h = (const void**)calloc(1, nbytes);
  dev = xb_rt_scratch(nbytes);
  if (h == NULL || dev == NULL) { free(h); return NULL; }
  for (r = 0; r < br; ++r) h[r] = xb_stage_in(((const void* const*)arr)[r], bytes, staged);
  xb_rt_upload(dev, h, nbytes);
  xb_rt_sync();                      /* h is pageable: make sure the upload consumed it */
  free(h);
  *staged = 1;
  return dev;
}

/* stages the side operands xb_gemm_sides names for one call of br blocks into one->a_s, b_s, c_s and a_q (NULL where the call has none):
 * the only code that knows their byte extents. An MXBF8 C's scales are written by the kernel: a pageable c.tertiary gets a device block
 * that xb_invoke_gemm copies back. */
static void xb_stage_sides(const xb_gemm_desc* d, const libxsmm_gemm_param* p, unsigned long long br, xb_gemm_rec* one, int* staged) {
  const int sides = xb_gemm_sides(d);
  if (sides == 0) return;
  switch (d->path) {
    case P_DQ:       /* a.tertiary: m row scales (f32 next to a bf16 B, else f16); int4: a.quaternary, m f16 zero points. One set for every r. */
      one->a_s = xb_stage_in(p->a.tertiary, (size_t)d->m * (xb_dq_form(d) == XB_DQ_I8_BF16 ? 4 : 2), staged);
      if (sides & XB_SIDE_A_Q) one->a_q = xb_stage_in(p->a.quaternary, (size_t)d->m * 2, staged);
      break;
    case P_LOWBIT: { /* MXFP4: a.tertiary, E8M0 bytes [k/32][lda]; b.tertiary, f32 [n][ldb/32]; block r's as in xb_gemm_simt */
      const size_t ea = (size_t)(d->k / 32 - 1) * d->lda + (size_t)d->m, eb = ((size_t)(d->n - 1) * (size_t)(d->ldb / 32) + (size_t)(d->k / 32)) * 4;
      if (d->br_type == 1) {
        one->a_s = xb_stage_ptr_array(p->a.tertiary, br, ea, staged);
        one->b_s = xb_stage_ptr_array(p->b.tertiary, br, eb, staged);
      } else {
        size_t span_sa = ea, span_sb = eb;
        unsigned long long r;
        if (d->br_type == 3 && br > 0) { span_sa += (size_t)(br - 1) * (size_t)((d->br_stride_a * 2) / 32); span_sb += (size_t)(br - 1) * (size_t)(d->br_stride_b / 32) * 4; }
        if (d->br_type == 2) for (r = 0; r < br; ++r) {
          const long long oa = (((const long long*)p->a.secondary)[r] * 2) / 32, ob = ((const long long*)p->b.secondary)[r] / 32;
          if (oa > 0 && ea + (size_t)oa > span_sa) span_sa = ea + (size_t)oa;
          if (ob > 0 && eb + (size_t)ob * 4 > span_sb) span_sb = eb + (size_t)ob * 4;
        }
        one->a_s = xb_stage_in(p->a.tertiary, span_sa, staged);
        one->b_s = xb_stage_in(p->b.tertiary, span_sb, staged);
      }
      break;
    }
    case P_I4_I32: { /* int4 A x 8-bit B: a.quaternary, one zero-point byte per row (and per reduce step) */
      const size_t zb = (size_t)d->m + ((d->br_type == 3 && br > 0) ? (size_t)(br - 1) * (size_t)((d->br_stride_a * 2) / d->k) : 0);
      one->a_q = xb_stage_in(p->a.quaternary, zb, staged);
      break;
    }
    default:         /* MX fp8, E8M0 block scales: a.tertiary [br][k/32][lda], b.tertiary [br][k/32][ldb] and, for an MXBF8 C, c.tertiary [n][ldc/32] */
      one->a_s = xb_stage_in(p->a.tertiary, xb_extent_mx_scales(d, br, d->lda, d->m), staged);
      one->b_s = xb_stage_in(p->b.tertiary, xb_extent_mx_scales(d, br, d->ldb, d->n), staged);
      if (sides & XB_SIDE_C_S) {
        *staged = 1;                   /* the f32 image lives in the scratch arena until the caller's sync */
        one->c_s = (p->c.tertiary != NULL && xb_rt_ptr_kind(p->c.tertiary) == 0) ? xb_rt_scratch((size_t)(d->n - 1) * (d->ldc / 32) + (size_t)(d->m / 32))
                                                                                 : p->c.tertiary;
      }
  }
}

static int xb_run_gemm_launch(const xb_gemm_launch* L) {
  if (L->d.backend != LIBXSMM_B200_BACKEND_TCGEN05) return xb_gemm_simt_launch(L);
  return xb_gemm_ts_supported(&L->d) ? xb_gemm_ts_launch(L) : xb_gemm_tc_launch(L);
}

static void xb_invoke_gemm(const xb_slot* s, const libxsmm_gemm_param* p) {
  const xb_gemm_desc* d = &s->u.gemm;
  const size_t tsa = libxsmm_typesize((libxsmm_datatype)d->ta), tsb = libxsmm_typesize((libxsmm_datatype)d->tb);
  const size_t tsc = libxsmm_typesize((libxsmm_datatype)d->tc);
  const int vnni_c = (d->flags & LIBXSMM_GEMM_FLAG_VNNI_C) != 0 && tsc == 2;   /* packs the whole ldc x n image, padding rows included */
  const size_t ext_a = xb_extent_a(d) * tsa, ext_b = xb_extent_b(d) * tsb, ext_c = (vnni_c ? (size_t)d->n * d->ldc : ((size_t)(d->n - 1) * d->ldc + d->m)) * tsc;
  const unsigned long long br = (d->br_type != 0 && p->op.tertiary != NULL) ? *(const unsigned long long*)p->op.tertiary : 1ull;
  xb_gemm_launch L;
  const int sides = xb_gemm_sides(d);
  xb_copyback cb, cb_mask; int staged = 0, need_cb = 0, need_cb_mask = 0;
  memset(&L, 0, sizeof(L)); memset(&cb, 0, sizeof(cb)); memset(&cb_mask, 0, sizeof(cb_mask));
  L.d = *d; L.count = 1;
  L.one.br = br;
  if (d->br_type != 0 && br == 0) {  /* nothing to reduce: reference still zeroes C for beta=0 */ }
  /* A and B */
  if (d->br_type == 1) {             /* arrays of br pointers, readable on the host unless device memory */
    if (xb_rt_ptr_kind(p->a.primary) == 1) { L.one.a = p->a.primary; L.one.b = p->b.primary; }
    else {
      const void** ha = (const void**)malloc(2 * (size_t)(br ? br : 1) * sizeof(void*));
      const void** hb = ha + (br ? br : 1);
      void* dev = xb_rt_scratch(2 * (size_t)(br ? br : 1) * sizeof(void*));
      unsigned long long r;
      if (ha == NULL || dev == NULL) { free(ha); xb_rt_note_error(2, "invoke_gemm: out of memory"); return; }
      for (r = 0; r < br; ++r) {
        ha[r] = xb_stage_in(((void* const*)p->a.primary)[r], ext_a, &staged);
        hb[r] = xb_stage_in(((void* const*)p->b.primary)[r], ext_b, &staged);
      }
      xb_rt_upload(dev, ha, 2 * (size_t)(br ? br : 1) * sizeof(void*));
      xb_rt_sync();                  /* ha is pageable: make sure the upload consumed it */
      free(ha);
      L.one.a = dev; L.one.b = (const char*)dev + (size_t)(br ? br : 1) * sizeof(void*);
      staged = 1;
    }
  } else {
    size_t span_a = ext_a, span_b = ext_b;
    if (d->br_type == 3 && br > 0) { span_a += (size_t)(br - 1) * (size_t)d->br_stride_a; span_b += (size_t)(br - 1) * (size_t)d->br_stride_b; }
    if (d->br_type == 2 && br > 0) {
      const long long* oa = (const long long*)p->a.secondary; const long long* ob = (const long long*)p->b.secondary;
      long long ma = 0, mb = 0; unsigned long long r;
      void* dev = xb_rt_scratch(2 * (size_t)br * sizeof(long long));
      if (dev == NULL) return;
      for (r = 0; r < br; ++r) { if (oa[r] > ma) ma = oa[r]; if (ob[r] > mb) mb = ob[r]; }
      span_a += (size_t)ma; span_b += (size_t)mb;
      xb_rt_upload(dev, oa, (size_t)br * sizeof(long long));
      xb_rt_upload((char*)dev + (size_t)br * sizeof(long long), ob, (size_t)br * sizeof(long long));
      L.one.a_aux = dev; L.one.b_aux = (const char*)dev + (size_t)br * sizeof(long long);
      staged = 1;
    }
    if ((d->flags & LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK) != 0) {   /* a.secondary: bitmap; A holds one element per set bit */
      const size_t bbytes = ((size_t)d->m * d->k + 7) / 8;
      if (p->a.secondary == NULL) { xb_rt_note_error(2, "invoke_gemm: bitmap missing (a.secondary)"); xb_rt_scratch_reset(); return; }
      if (xb_rt_ptr_kind(p->a.secondary) != 1) {   /* host-readable bitmap: count the stored elements */
        const unsigned char* bm = (const unsigned char*)p->a.secondary; size_t nz = 0, q;
        for (q = 0; q < bbytes; ++q) nz += (size_t)__builtin_popcount(bm[q]);
        span_a = nz * tsa;
      } else if (xb_rt_ptr_kind(p->a.primary) == 0) { xb_rt_note_error(2, "invoke_gemm: device bitmap with host A"); xb_rt_scratch_reset(); return; }
      L.one.a_q = xb_stage_in(p->a.secondary, bbytes, &staged);
    }
    L.one.a = xb_stage_in(p->a.primary, span_a ? span_a : 1, &staged);
    L.one.b = xb_stage_in(p->b.primary, span_b, &staged);
  }
  xb_stage_sides(d, p, br, &L.one, &staged);
  if (xb_gemm_rec_lacks(&L.one, sides)) {
    xb_rt_note_error(1, "invoke_gemm: side operand missing (scales in a/b/c.tertiary, zero points in a.quaternary)"); xb_rt_scratch_reset(); return;
  }
  /* C: staged copy is seeded from the host whenever old contents can survive (beta=1 or ldc>m) */
  if (p->c.primary != NULL && xb_rt_ptr_kind(p->c.primary) == 0) {
    void* dc = xb_rt_scratch(ext_c);
    if (dc == NULL) return;
    if ((d->flags & LIBXSMM_GEMM_FLAG_BETA_0) == 0 || d->ldc != d->m || d->fuse_colbias == 0) xb_rt_upload(dc, p->c.primary, ext_c);
    cb.host = p->c.primary; cb.dev = dc; cb.bytes = ext_c; need_cb = 1; staged = 1;
    L.one.c = dc;
  } else L.one.c = p->c.primary;
  if (d->path == P_I8_F32 && p->c.tertiary != NULL) L.one.scf = *(const float*)p->c.tertiary;
  if (s->kind == XB_KIND_GEMM_EXT && (d->fuse_colbias != 0 || d->cp_op != 0)) {   /* d.primary: bias column; c.secondary: ReLU bitmask */
    const libxsmm_gemm_ext_param* pe = (const libxsmm_gemm_ext_param*)p;
    if (d->fuse_colbias != 0) {
      L.one.d = xb_stage_in(pe->d.primary, (size_t)d->m * tsc, &staged);
      if (L.one.d == NULL) { xb_rt_note_error(2, "invoke_gemm_ext: bias column missing"); xb_rt_scratch_reset(); return; }
    }
    if ((d->cp_flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0 && pe->c.secondary != NULL) {
      const size_t mbytes = (size_t)LIBXSMM_UP(d->ldc, 16) / 8 * (size_t)d->n;
      if (xb_rt_ptr_kind(pe->c.secondary) == 0) {
        void* dm = xb_rt_scratch(mbytes);
        if (dm == NULL) return;
        xb_rt_upload(dm, pe->c.secondary, mbytes);           /* bits of padding rows survive */
        cb_mask.host = pe->c.secondary; cb_mask.dev = dm; cb_mask.bytes = mbytes; need_cb_mask = 1; staged = 1;
        L.one.c_aux = dm;
      } else L.one.c_aux = pe->c.secondary;
    }
  }
  if (0 != xb_run_gemm_launch(&L)) { xb_rt_scratch_reset(); return; }
  if (vnni_c) {   /* C re-packed norm -> VNNI2 through a copy (reference :2803-2815) */
    void* copy = xb_rt_scratch(ext_c);
    xb_meltw_desc md; xb_meltw_args ma;
    if (copy == NULL) { xb_rt_scratch_reset(); return; }
    xb_rt_memcpy_async(copy, L.one.c, ext_c);
    memset(&md, 0, sizeof(md)); memset(&ma, 0, sizeof(ma));
    md.op_class = LIBXSMM_MELTW_OPERATION_UNARY; md.op = LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2; md.m = d->m; md.n = d->n;
    md.ldi = d->ldc; md.ldo = d->ldc; md.t_in0 = md.t_out = md.t_comp = d->tc; md.t_in1 = md.t_in2 = LIBXSMM_DATATYPE_UNSUPPORTED;
    ma.in0 = copy; ma.out = L.one.c; ma.alpha = 1.0f;
    if (0 != xb_meltw_launch(&md, &ma)) { xb_rt_scratch_reset(); return; }
    staged = 1;
  }
  if (need_cb) {
    /* only the m x n block this call owns goes back: callers update row blocks of ONE host C from several threads (ldc > m), and the
     * contiguous span would carry the neighbours' rows back stale over their results. VNNI-packed C is re-packed as a whole ldc x n image. */
    if (vnni_c) xb_rt_memcpy_async(cb.host, cb.dev, cb.bytes);
    else xb_rt_memcpy2d_async(cb.host, cb.dev, (size_t)d->ldc * tsc, (size_t)d->m * tsc, (size_t)d->n);
  }
  if (need_cb_mask) xb_rt_memcpy_async(cb_mask.host, cb_mask.dev, cb_mask.bytes);
  if ((sides & XB_SIDE_C_S) && L.one.c_s != p->c.tertiary) xb_rt_memcpy2d_async(p->c.tertiary, L.one.c_s, (size_t)(d->ldc / 32), (size_t)(d->m / 32), (size_t)d->n);   /* the m/32 scale bytes of each column */
  if (staged || xb_rt_blocking()) { xb_rt_sync(); xb_rt_scratch_reset(); }
}

/* ---- BLAS-style entry points (reference src/libxsmm_main.c:3933-3949) ----------------------------------------------------------
 * LIBXSMM_XGEMM (reference src/libxsmm_main.h:215-240) with its quirks, so that a relinked caller gets the reference's numbers rather
 * than BLAS's: alpha is never read; beta only chooses between BETA_0 (beta == 0) and accumulate (any other value, 0.5 included, acts
 * as 1; NULL means LIBXSMM_BETA); k defaults to m and n to k; lda defaults to m (k under TRANS_A), ldb to k (n under TRANS_B), ldc to
 * m, and every leading dimension is at least 1. A shape the descriptor rejects prints "LIBXSMM_GEMM failed" and leaves C alone. */
static void xb_blas_gemm(libxsmm_datatype type, const char* transa, const char* transb,
  const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const void* a, const libxsmm_blasint* lda, const void* b, const libxsmm_blasint* ldb,
  const void* beta, void* c, const libxsmm_blasint* ldc)
{
  const int beta0 = (beta != NULL) && ((type == LIBXSMM_DATATYPE_F64) ? (*(const double*)beta == 0) : (*(const float*)beta == 0));
  const libxsmm_bitfield flags = LIBXSMM_GEMM_PFLAGS(transa, transb, LIBXSMM_FLAGS) | (beta0 ? LIBXSMM_GEMM_FLAG_BETA_0 : 0);
  const libxsmm_blasint* kk = (k != NULL) ? k : m;
  const libxsmm_blasint* nn = (n != NULL) ? n : kk;
  const libxsmm_blasint ld_a = LIBXSMM_MAX((lda != NULL) ? *lda : *((flags & LIBXSMM_GEMM_FLAG_TRANS_A) == 0 ? m : kk), 1);
  const libxsmm_blasint ld_b = LIBXSMM_MAX((ldb != NULL) ? *ldb : *((flags & LIBXSMM_GEMM_FLAG_TRANS_B) == 0 ? kk : nn), 1);
  const libxsmm_blasint ld_c = LIBXSMM_MAX((ldc != NULL) ? *ldc : *m, 1);
  const libxsmm_gemm_shape shape = libxsmm_create_gemm_shape(*m, *nn, *kk, ld_a, ld_b, ld_c, type, type, type, type);
  const libxsmm_gemmfunction kernel = xb_dispatch_gemm_common(&shape, flags, LIBXSMM_PREFETCH, NULL);
  if (kernel != NULL) {
    libxsmm_gemm_param p;
    memset(&p, 0, sizeof(p));
    p.a.primary = (void*)(uintptr_t)a; p.b.primary = (void*)(uintptr_t)b; p.c.primary = c;
    xb_invoke_gemm(xb_slot_of((const void*)kernel), &p);
  }
  else printf("LIBXSMM_GEMM failed\n");
}

LIBXSMM_API void libxsmm_dgemm(const char* transa, const char* transb,
  const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const double* alpha, const double* a, const libxsmm_blasint* lda,
  const double* b, const libxsmm_blasint* ldb,
  const double* beta, double* c, const libxsmm_blasint* ldc)
{
  (void)alpha;
  xb_blas_gemm(LIBXSMM_DATATYPE_F64, transa, transb, m, n, k, a, lda, b, ldb, beta, c, ldc);
}

LIBXSMM_API void libxsmm_sgemm(const char* transa, const char* transb,
  const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const float* alpha, const float* a, const libxsmm_blasint* lda,
  const float* b, const libxsmm_blasint* ldb,
  const float* beta, float* c, const libxsmm_blasint* ldc)
{
  (void)alpha;
  xb_blas_gemm(LIBXSMM_DATATYPE_F32, transa, transb, m, n, k, a, lda, b, ldb, beta, c, ldc);
}

/* Fortran-77 symbols (reference src/libxsmm_main.c:4313-4340, LIBXSMM_FSYMBOL): every argument by reference already */
LIBXSMM_API void libxsmm_dgemm_(const char* transa, const char* transb,
  const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const double* alpha, const double* a, const libxsmm_blasint* lda,
  const double* b, const libxsmm_blasint* ldb,
  const double* beta, double* c, const libxsmm_blasint* ldc)
{
  libxsmm_dgemm(transa, transb, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}

LIBXSMM_API void libxsmm_sgemm_(const char* transa, const char* transb,
  const libxsmm_blasint* m, const libxsmm_blasint* n, const libxsmm_blasint* k,
  const float* alpha, const float* a, const libxsmm_blasint* lda,
  const float* b, const libxsmm_blasint* ldb,
  const float* beta, float* c, const libxsmm_blasint* ldc)
{
  libxsmm_sgemm(transa, transb, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}

/* ---- batch entry points -------------------------------------------------------------------------- */
static const xb_slot* xb_gemm_slot(const void* kernel) {
  const xb_slot* s = xb_slot_of(kernel);
  return (s != NULL && (s->kind == XB_KIND_GEMM || s->kind == XB_KIND_GEMM_EXT)) ? s : NULL;
}

/* 1 if a batch entry point cannot run this handle as a single call would: a fused handle's bias column and ReLU bit mask are
 * per-call operands (libxsmm_gemm_ext_param) that no batch form carries, VNNI-packed C is re-packed by a pass after a single
 * call only, the strided forms have no argument struct for the int8 -> f32 scale (c.tertiary) or for side operands
 * (xb_gemm_sides: libxsmm_b200_gemm_batch_strided_scaled takes scales), and the per-tile records carry no MX fp8 block scales. */
static int xb_batch_refused(const xb_gemm_desc* d, int strided) {
  if (d->fuse_colbias != 0 || (d->flags & LIBXSMM_GEMM_FLAG_VNNI_C) != 0) return 1;
  if (strided ? xb_gemm_sides(d) != 0 : d->path == P_MX8) return 1;
  if (d->cp_op == LIBXSMM_MELTW_TYPE_UNARY_RELU && (d->cp_flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0) return 1;
  return (strided && d->path == P_I8_F32) ? 1 : 0;
}

/* host-resident strided batch: chunked H2D -> kernel -> D2H through device scratch */
static int xb_gemm_batch_strided_host(const xb_slot* s, const void* a, const void* b, void* c,
  long long sa, long long sb, long long sc, unsigned long long br, long long count);

LIBXSMM_API int libxsmm_b200_gemm_batch_strided(libxsmm_gemmfunction kernel, const void* a, const void* b, void* c,
  long long stride_a, long long stride_b, long long stride_c, unsigned long long br_count, long long count)
{
  const xb_slot* s = xb_gemm_slot((const void*)kernel);
  xb_gemm_launch L;
  int rc;
  if (s == NULL || count < 0) return -1;
  if (xb_batch_refused(&s->u.gemm, 1)) return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
  if (s->u.gemm.br_type == 1 || s->u.gemm.br_type == 2) return -2;   /* address / offset mode need per-tile arrays: use libxsmm_b200_gemm_batch */
  if (count == 0) return 0;
  {
    const int ka = xb_rt_ptr_kind(a), kb = xb_rt_ptr_kind(b), kc = xb_rt_ptr_kind(c);
    const char* zc = getenv("LIBXSMM_B200_ZEROCOPY");
    const int zero_copy = (zc != NULL && zc[0] == '1');       /* pinned memory is device-accessible: optional in-place access */
    const int host = (ka == 0 || kb == 0 || kc == 0) || (!zero_copy && (ka == 3 || kb == 3 || kc == 3));
    if (host) {
      if ((ka == 0 || ka == 3) && (kb == 0 || kb == 3) && (kc == 0 || kc == 3)) {
        return xb_gemm_batch_strided_host(s, a, b, c, stride_a, stride_b, stride_c, br_count, count);
      }
      if (ka == 0 || kb == 0 || kc == 0) return -4;            /* mixed pageable-host / device operands: not supported in one call */
    }
  }
  memset(&L, 0, sizeof(L));
  L.d = s->u.gemm; L.count = count;
  L.a = a; L.b = b; L.c = c; L.tile_stride_a = stride_a; L.tile_stride_b = stride_b; L.tile_stride_c = stride_c;
  L.br = (s->u.gemm.br_type == 0) ? 1ull : br_count;
  rc = xb_run_gemm_launch(&L);
  if (rc == 0 && xb_rt_blocking()) rc = xb_rt_sync();
  return rc;
}

#define XB_MX_IMAGE_BYTES (64ll << 20)   /* f32 image of an MXBF8-C batch: scratch per chunk */

LIBXSMM_API int libxsmm_b200_gemm_batch_strided_scaled(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  const void* scf_a, const void* scf_b, void* scf_c, long long stride_scf_a, long long stride_scf_b, long long stride_scf_c,
  unsigned long long br_count, long long count)
{
  const xb_slot* s = xb_gemm_slot((const void*)kernel);
  xb_gemm_launch L;
  int rc, sides;
  if (s == NULL || count < 0 || s->kind != XB_KIND_GEMM) return -1;
  /* handles with scales and no zero points (those need libxsmm_b200_gemm_batch); tile t's are scf_x + t*stride_scf_x */
  sides = xb_gemm_sides(&s->u.gemm);
  if (sides == 0 || (sides & XB_SIDE_A_Q) != 0) return -1;
  if (count == 0) return 0;
  memset(&L, 0, sizeof(L));
  L.d = s->u.gemm;
  L.tile_stride_a = stride_a; L.tile_stride_b = stride_b; L.tile_stride_c = stride_c;
  L.br = (L.d.br_type == 0) ? 1ull : br_count;
  if (sides & XB_SIDE_A_S) { L.one.a_s = scf_a; L.tile_stride_as = stride_scf_a; }
  if (sides & XB_SIDE_B_S) { L.one.b_s = scf_b; L.tile_stride_bs = stride_scf_b; }
  if (sides & XB_SIDE_C_S) { L.one.c_s = scf_c; L.tile_stride_cs = stride_scf_c; }
  if (a == NULL || b == NULL || c == NULL || xb_gemm_rec_lacks(&L.one, sides)) return -1;
  if (L.d.br_type == 1 || L.d.br_type == 2) return -2;   /* per-tile arrays: libxsmm_b200_gemm_batch */
  if (xb_rt_ptr_kind(a) == 0 || xb_rt_ptr_kind(b) == 0 || xb_rt_ptr_kind(c) == 0 || (L.one.a_s != NULL && xb_rt_ptr_kind(L.one.a_s) == 0)
   || (L.one.b_s != NULL && xb_rt_ptr_kind(L.one.b_s) == 0) || (L.one.c_s != NULL && xb_rt_ptr_kind(L.one.c_s) == 0)) return -4;   /* device-accessible operands only */
  if ((sides & XB_SIDE_C_S) == 0) {
    L.count = count; L.a = a; L.b = b; L.c = c;
    rc = xb_run_gemm_launch(&L);
    if (rc == 0 && xb_rt_blocking()) rc = xb_rt_sync();
    return rc;
  }
  {
    /* MXBF8 C: the product goes through an f32 image of m*n*4 bytes per tile in the thread's scratch arena, which keeps its size
     * once grown. The batch runs in chunks of at most XB_MX_IMAGE_BYTES of image, each synchronised before the arena is reused. */
    const long long per_tile = (long long)L.d.m * L.d.n * 4;
    const long long chunk = (per_tile < XB_MX_IMAGE_BYTES) ? XB_MX_IMAGE_BYTES / per_tile : 1;
    long long t0;
    rc = 0;
    for (t0 = 0; t0 < count && rc == 0; t0 += chunk) {
      int rs;
      L.count = (count - t0 < chunk) ? (count - t0) : chunk;
      L.a = (const char*)a + t0 * stride_a; L.b = (const char*)b + t0 * stride_b; L.c = (char*)c + t0 * stride_c;
      L.one.a_s = (const char*)scf_a + t0 * stride_scf_a; L.one.b_s = (const char*)scf_b + t0 * stride_scf_b;
      L.one.c_s = (char*)scf_c + t0 * stride_scf_c;
      rc = xb_run_gemm_launch(&L);
      rs = xb_rt_sync();
      if (rc == 0) rc = rs;
      xb_rt_scratch_reset();
    }
    return rc;
  }
}

/* ---- one process, several GPUs: the batch is the only shard axis (SURVEY.md 8e). Host-resident operands are cut into
 * `ndevices` contiguous ranges; one worker thread per device moves its range over its own PCIe link through the chunked copy
 * pipeline and runs the kernel there. Nothing is exchanged between devices; the results land in the caller's C. ---------- */
typedef struct xb_multi_job {
  libxsmm_gemmfunction kernel; const char* a; const char* b; char* c; long long sa, sb, sc, first, count; unsigned long long br; int device, rc;
} xb_multi_job;

static void* xb_multi_worker(void* arg) {
  xb_multi_job* j = (xb_multi_job*)arg;
  j->rc = xb_rt_set_device(j->device);
  if (j->rc == 0) {
    xb_rt_set_stream(NULL); xb_rt_set_blocking(1);
    j->rc = libxsmm_b200_gemm_batch_strided(j->kernel, j->a + j->first * j->sa, j->b + j->first * j->sb, j->c + j->first * j->sc,
                                            j->sa, j->sb, j->sc, j->br, j->count);
    xb_rt_scratch_reset();
  }
  return NULL;
}

LIBXSMM_API int libxsmm_b200_gemm_batch_strided_multi(libxsmm_gemmfunction kernel, const void* a, const void* b, void* c,
  long long stride_a, long long stride_b, long long stride_c, unsigned long long br_count, long long count, int ndevices)
{
  xb_multi_job jobs[64]; pthread_t th[64];
  int d, rc = 0, started = 0, prev_dev;
  const int avail = xb_rt_device_count();
  if (xb_gemm_slot((const void*)kernel) == NULL || count < 0 || ndevices <= 0) return -1;
  if (xb_batch_refused(&xb_gemm_slot((const void*)kernel)->u.gemm, 1)) return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
  if (ndevices > avail) ndevices = avail;
  if (ndevices > 64) ndevices = 64;
  if (ndevices <= 0) return -1;
  if (xb_rt_ptr_kind(a) == 1 || xb_rt_ptr_kind(b) == 1 || xb_rt_ptr_kind(c) == 1) return -4;   /* device memory belongs to one GPU: use the per-device call */
  prev_dev = xb_rt_current_device();
  for (d = 0; d < ndevices; ++d) {
    const long long base = count / ndevices, extra = count % ndevices;
    xb_multi_job* j = &jobs[d];
    j->kernel = kernel; j->a = (const char*)a; j->b = (const char*)b; j->c = (char*)c; j->sa = stride_a; j->sb = stride_b; j->sc = stride_c; j->br = br_count;
    j->first = d * base + (d < extra ? d : extra); j->count = base + (d < extra ? 1 : 0); j->device = d; j->rc = 0;
    if (j->count == 0) { th[d] = 0; continue; }
    if (0 != pthread_create(&th[d], NULL, xb_multi_worker, j)) { j->rc = -5; th[d] = 0; } else ++started;
  }
  for (d = 0; d < ndevices; ++d) { if (th[d] != 0) pthread_join(th[d], NULL); if (jobs[d].rc != 0 && rc == 0) rc = jobs[d].rc; }
  (void)started;
  xb_rt_set_device(prev_dev);
  return rc;
}

typedef struct xb_hostbatch {
  const xb_gemm_desc* d; const char* a; const char* b; char* c;
  long long sa, sb, sc, chunk, count; unsigned long long br;
  size_t fa, fb, fc; int copy_c_in;
} xb_hostbatch;

static void xb_hostbatch_describe(void* ctx, long long i, xb_pipe_chunk* ch) {
  const xb_hostbatch* h = (const xb_hostbatch*)ctx;
  const long long t0 = i * h->chunk, nt = (h->count - t0 < h->chunk) ? (h->count - t0) : h->chunk;
  ch->first = t0; ch->count = nt;
  ch->host_a = h->a + t0 * h->sa; ch->host_b = h->b + t0 * h->sb; ch->host_c = h->c + t0 * h->sc;
  ch->bytes_a = (size_t)(nt - 1) * (size_t)h->sa + h->fa; ch->bytes_b = (size_t)(nt - 1) * (size_t)h->sb + h->fb;
  ch->bytes_c = (size_t)(nt - 1) * (size_t)h->sc + h->fc; ch->copy_c_in = h->copy_c_in;
}

static int xb_hostbatch_launch(void* ctx, const xb_pipe_chunk* ch, void* da, void* db, void* dc) {
  const xb_hostbatch* h = (const xb_hostbatch*)ctx;
  xb_gemm_launch L;
  memset(&L, 0, sizeof(L));
  L.d = *h->d; L.count = ch->count; L.a = da; L.b = db; L.c = dc;
  L.tile_stride_a = h->sa; L.tile_stride_b = h->sb; L.tile_stride_c = h->sc; L.br = (h->d->br_type == 0) ? 1ull : h->br;
  return xb_run_gemm_launch(&L);
}

static int xb_gemm_batch_strided_host(const xb_slot* s, const void* a, const void* b, void* c,
  long long sa, long long sb, long long sc, unsigned long long br, long long count)
{
  /* the batch is cut into chunks that flow through xb_rt_pipeline: the copies of chunk i+1 (H2D) and of chunk i-1 (D2H)
   * overlap the kernel of chunk i. Every chunk is a dense range of tiles, which requires the tile strides to cover the
   * tile footprint (checked: positive strides). Returns when C is valid in host memory. */
  const xb_gemm_desc* d = &s->u.gemm;
  const size_t tsa = libxsmm_typesize((libxsmm_datatype)d->ta), tsb = libxsmm_typesize((libxsmm_datatype)d->tb);
  const size_t tsc = libxsmm_typesize((libxsmm_datatype)d->tc);
  xb_hostbatch h;
  long long nchunks;
  if (sa <= 0 || sb <= 0 || sc <= 0 || d->br_type == 2) return -3;
  memset(&h, 0, sizeof(h));
  h.d = d; h.a = (const char*)a; h.b = (const char*)b; h.c = (char*)c; h.sa = sa; h.sb = sb; h.sc = sc; h.br = br; h.count = count;
  h.fa = xb_extent_a(d) * tsa; h.fb = xb_extent_b(d) * tsb; h.fc = ((size_t)(d->n - 1) * d->ldc + d->m) * tsc;
  if (d->br_type == 3 && br > 0) { h.fa += (size_t)(br - 1) * (size_t)d->br_stride_a; h.fb += (size_t)(br - 1) * (size_t)d->br_stride_b; }
  h.copy_c_in = ((d->flags & LIBXSMM_GEMM_FLAG_BETA_0) == 0 || (size_t)sc != h.fc) ? 1 : 0;
  {
    const size_t per_tile = (size_t)sa + (size_t)sb + (size_t)sc;
    size_t budget = (size_t)128 << 20;            /* staging bytes per chunk: small enough to overlap, large enough to amortise launches */
    const char* e = getenv("LIBXSMM_B200_CHUNK_MB");
    if (e != NULL && atoi(e) > 0) budget = (size_t)atoi(e) << 20;
    h.chunk = (long long)(budget / (per_tile ? per_tile : 1));
    if (h.chunk < 1) h.chunk = 1;
    if (h.chunk > count) h.chunk = count;
  }
  nchunks = (count + h.chunk - 1) / h.chunk;
  return xb_rt_pipeline(nchunks, (size_t)(h.chunk - 1) * (size_t)sa + h.fa, (size_t)(h.chunk - 1) * (size_t)sb + h.fb,
                        (size_t)(h.chunk - 1) * (size_t)sc + h.fc, xb_hostbatch_describe, xb_hostbatch_launch, &h);
}

struct libxsmm_b200_gemm_plan {
  const xb_slot* slot;
  xb_gemm_rec* d_recs;       /* device */
  void* d_arrays;            /* device: per-tile pointer/offset arrays */
  long long count;
  /* address batch-reduce whose blocks form regular block-sets in a pool (base + set*set_stride + r*block_stride): served by the
   * tensor-core kernel with the set index as tensor-map coordinate; tiles are sorted by set pair so that two tiles sharing a B set
   * form one item (the reference calls the kernel once per tile, the order is free) */
  int pooled; xb_tc_pool pool; unsigned long long br; void* d_sets; void* d_cptrs;
};

static int xb_env_flag(const char* name, int fallback) { const char* e = getenv(name); return (e != NULL && *e != 0) ? (atoi(e) != 0) : fallback; }
typedef struct xb_pool_key { long long sa, sb; long long t; } xb_pool_key;
static int xb_pool_key_cmp(const void* x, const void* y) {      /* by set of B, then set of A: neighbours share B (pairing) and often A too */
  const xb_pool_key* a = (const xb_pool_key*)x; const xb_pool_key* b = (const xb_pool_key*)y;
  if (a->sb != b->sb) return (a->sb < b->sb) ? -1 : 1;
  if (a->sa != b->sa) return (a->sa < b->sa) ? -1 : 1;
  return (a->t < b->t) ? -1 : (a->t > b->t);
}
static long long xb_gcd_ll(long long a, long long b) { while (b != 0) { const long long c = a % b; a = b; b = c; } return a; }

/* returns 1 and fills the plan if the address-mode batch is a regular pool the tensor-core kernel can walk */
static int xb_plan_try_pool(libxsmm_b200_gemm_plan* plan, const xb_slot* s, const libxsmm_gemm_param* params, long long count) {
  const xb_gemm_desc* d = &s->u.gemm;
  unsigned long long br; long long t, blk_a = 0, blk_b = 0, set_a = 0, set_b = 0; unsigned long long r;
  uintptr_t base_a = (uintptr_t)-1, base_b = (uintptr_t)-1;
  xb_pool_key* keys; int* sets; void** cptrs; int ok = 1;
  long long items = 0;
  const int pair = (d->m <= 64 && count > 1 && xb_env_flag("LIBXSMM_B200_TC_PAIR", 1)) ? 1 : 0;   /* two 64-row tiles per M=128 instruction */
  const int offs_mode = (d->br_type == 2);       /* OFFSET batch-reduce: block r = a.primary + a.secondary[r]; same regularity test */
#define XB_POOL_BLK(ARG, R) (offs_mode ? (uintptr_t)(ARG).primary + (uintptr_t)((const unsigned long long*)(ARG).secondary)[R] \
                                       : (uintptr_t)((const void* const*)(ARG).primary)[R])
  if ((d->br_type != 1 && d->br_type != 2) || g_force_simt || !xb_gemm_tc_shape_ok(d) || count > 0x7fffffffll) return 0;
  if (params[0].op.tertiary == NULL) return 0;
  br = *(const unsigned long long*)params[0].op.tertiary;
  if (br == 0 || br > 4096) return 0;
  for (t = 0; t < count && ok; ++t) {          /* pass 1: common block stride, lowest address */
    const libxsmm_gemm_param* p = &params[t];
    const void* pa = offs_mode ? p->a.secondary : p->a.primary; const void* pb = offs_mode ? p->b.secondary : p->b.primary;   /* the host-side index arrays */
    if (p->op.tertiary == NULL || *(const unsigned long long*)p->op.tertiary != br || pa == NULL || pb == NULL || p->a.primary == NULL || p->b.primary == NULL
     || xb_rt_ptr_kind(pa) == 1 || xb_rt_ptr_kind(pb) == 1 || xb_rt_ptr_kind(p->c.primary) == 0) { ok = 0; break; }
    for (r = 1; r < br; ++r) {
      const long long da = (long long)(XB_POOL_BLK(p->a, r) - XB_POOL_BLK(p->a, r - 1)), db = (long long)(XB_POOL_BLK(p->b, r) - XB_POOL_BLK(p->b, r - 1));
      if (blk_a == 0) { blk_a = da; blk_b = db; }
      if (da != blk_a || db != blk_b || da <= 0 || db <= 0 || (da % 16) != 0 || (db % 16) != 0) { ok = 0; break; }
    }
    if (XB_POOL_BLK(p->a, 0) < base_a) base_a = XB_POOL_BLK(p->a, 0);
    if (XB_POOL_BLK(p->b, 0) < base_b) base_b = XB_POOL_BLK(p->b, 0);
  }
  if (!ok || (base_a & 15) != 0 || (base_b & 15) != 0) return 0;
  if (br == 1) { blk_a = 16; blk_b = 16; }
  for (t = 0; t < count; ++t) {                /* pass 2: set stride = gcd of the set offsets */
    set_a = xb_gcd_ll(set_a, (long long)(XB_POOL_BLK(params[t].a, 0) - base_a));
    set_b = xb_gcd_ll(set_b, (long long)(XB_POOL_BLK(params[t].b, 0) - base_b));
  }
  if (set_a == 0) set_a = 16;
  if (set_b == 0) set_b = 16;
  if ((set_a % 16) != 0 || (set_b % 16) != 0) return 0;
  keys = (xb_pool_key*)malloc((size_t)count * sizeof(*keys)); sets = (int*)malloc((size_t)count * 4 * sizeof(int)); cptrs = (void**)malloc((size_t)count * 2 * sizeof(void*));
  if (keys == NULL || sets == NULL || cptrs == NULL) { free(keys); free(sets); free(cptrs); return 0; }
  plan->pool.nsets_a = plan->pool.nsets_b = 1;
  for (t = 0; t < count; ++t) {
    keys[t].sa = (long long)(XB_POOL_BLK(params[t].a, 0) - base_a) / set_a;
    keys[t].sb = (long long)(XB_POOL_BLK(params[t].b, 0) - base_b) / set_b;
    keys[t].t = t;
    if (keys[t].sa >= 0x7fffffffll || keys[t].sb >= 0x7fffffffll) ok = 0;
    if (keys[t].sa + 1 > plan->pool.nsets_a) plan->pool.nsets_a = keys[t].sa + 1;
    if (keys[t].sb + 1 > plan->pool.nsets_b) plan->pool.nsets_b = keys[t].sb + 1;
  }
  if (ok) {
    qsort(keys, (size_t)count, sizeof(*keys), xb_pool_key_cmp);
    /* items {set A, set A of the second tile, set B, 0}: in pair mode two neighbours with the same B set form one item (the
     * kernel stacks them into one M=128 instruction); a tile without such a neighbour travels alone (second C pointer NULL) */
    for (t = 0; t < count; ++items) {
      int* it = sets + 4 * items;
      const int two = (pair && t + 1 < count && keys[t + 1].sb == keys[t].sb) ? 1 : 0;
      it[0] = (int)keys[t].sa; it[1] = (int)keys[t + two].sa; it[2] = (int)keys[t].sb; it[3] = 0;
      if (pair) { cptrs[2 * items] = params[keys[t].t].c.primary; cptrs[2 * items + 1] = two ? params[keys[t + 1].t].c.primary : NULL; }
      else cptrs[items] = params[keys[t].t].c.primary;
      t += 1 + two;
    }
    plan->d_sets = xb_rt_device_malloc((size_t)items * 4 * sizeof(int)); plan->d_cptrs = xb_rt_device_malloc((size_t)items * (pair ? 2 : 1) * sizeof(void*));
    if (plan->d_sets == NULL || plan->d_cptrs == NULL || 0 != xb_rt_memcpy(plan->d_sets, sets, (size_t)items * 4 * sizeof(int))
     || 0 != xb_rt_memcpy(plan->d_cptrs, cptrs, (size_t)items * (pair ? 2 : 1) * sizeof(void*))) { xb_rt_device_free(plan->d_sets); xb_rt_device_free(plan->d_cptrs); plan->d_sets = plan->d_cptrs = NULL; ok = 0; }
  }
  free(keys); free(sets); free(cptrs);
  if (!ok) return 0;
  plan->pool.base_a = (const void*)base_a; plan->pool.base_b = (const void*)base_b; plan->pool.blk_a = blk_a; plan->pool.blk_b = blk_b;
  plan->pool.set_a = set_a; plan->pool.set_b = set_b; plan->pool.sets = plan->d_sets; plan->pool.cptrs = plan->d_cptrs; plan->pool.pair = pair;
  plan->pooled = 1; plan->br = br; plan->slot = s; plan->count = items;        /* the unit the kernel walks */
#undef XB_POOL_BLK
  return 1;
}

/* the side operands `sides` names in one call's argument struct, into the record fields the kernels read */
static void xb_param_sides(xb_gemm_rec* r, const libxsmm_gemm_param* p, int sides) {
  if (sides & XB_SIDE_A_S) r->a_s = p->a.tertiary;
  if (sides & XB_SIDE_B_S) r->b_s = p->b.tertiary;
  if (sides & XB_SIDE_C_S) r->c_s = p->c.tertiary;
  if (sides & XB_SIDE_A_Q) r->a_q = p->a.quaternary;
}

/* the per-tile records of a batch: libxsmm_b200_gemm_batch and libxsmm_b200_gemm_plan_create */
static libxsmm_b200_gemm_plan* xb_plan_make(const xb_slot* s, const libxsmm_gemm_param* params, long long count) {
  libxsmm_b200_gemm_plan* plan;
  xb_gemm_rec* recs;
  char* arrays = NULL; size_t arrays_bytes = 0, off = 0;
  long long t;
  int mx_arrays, sides;
  if (s == NULL || params == NULL || count <= 0 || xb_batch_refused(&s->u.gemm, 0)) return NULL;
  sides = xb_gemm_sides(&s->u.gemm);
  mx_arrays = (s->u.gemm.path == P_LOWBIT && (sides & XB_SIDE_B_S) != 0);   /* MXFP4 x I8 */
  for (t = 0; t < count && sides != 0; ++t) {   /* every tile brings each side operand of the handle */
    xb_gemm_rec r;
    memset(&r, 0, sizeof(r));
    xb_param_sides(&r, &params[t], sides);
    if (xb_gemm_rec_lacks(&r, sides)) return NULL;
  }
  plan = (libxsmm_b200_gemm_plan*)calloc(1, sizeof(*plan));
  if (plan != NULL && xb_plan_try_pool(plan, s, params, count)) return plan;
  recs = (xb_gemm_rec*)calloc((size_t)count, sizeof(xb_gemm_rec));
  if (plan == NULL || recs == NULL) { free(plan); free(recs); return NULL; }
  /* pass 1: size of the per-tile index arrays (address: 2*br pointers, offset: 2*br offsets) */
  if (s->u.gemm.br_type == 1 || s->u.gemm.br_type == 2) {
    for (t = 0; t < count; ++t) {
      const unsigned long long br = *(const unsigned long long*)params[t].op.tertiary;
      if (xb_rt_ptr_kind(params[t].a.primary) != 1 || s->u.gemm.br_type == 2) arrays_bytes += 2 * (size_t)br * 8;
      if (s->u.gemm.br_type == 1 && mx_arrays) {   /* MXFP4: the scale pointer arrays, copied alike */
        if (xb_rt_ptr_kind(params[t].a.tertiary) != 1) arrays_bytes += (size_t)br * 8;
        if (xb_rt_ptr_kind(params[t].b.tertiary) != 1) arrays_bytes += (size_t)br * 8;
      }
    }
    if (arrays_bytes) {
      arrays = (char*)malloc(arrays_bytes);
      plan->d_arrays = xb_rt_device_malloc(arrays_bytes);
      if (arrays == NULL || plan->d_arrays == NULL) { free(arrays); free(recs); xb_rt_device_free(plan->d_arrays); free(plan); return NULL; }
    }
  }
  for (t = 0; t < count; ++t) {
    const libxsmm_gemm_param* p = &params[t];
    xb_gemm_rec* r = &recs[t];
    r->br = (s->u.gemm.br_type != 0 && p->op.tertiary != NULL) ? *(const unsigned long long*)p->op.tertiary : 1ull;
    r->a = p->a.primary; r->b = p->b.primary; r->c = p->c.primary;
    if (s->u.gemm.br_type == 1 && xb_rt_ptr_kind(p->a.primary) != 1) {
      memcpy(arrays + off, p->a.primary, (size_t)r->br * 8); r->a = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
      memcpy(arrays + off, p->b.primary, (size_t)r->br * 8); r->b = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
    } else if (s->u.gemm.br_type == 2) {
      memcpy(arrays + off, p->a.secondary, (size_t)r->br * 8); r->a_aux = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
      memcpy(arrays + off, p->b.secondary, (size_t)r->br * 8); r->b_aux = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
    }
    xb_param_sides(r, p, sides);
    if (mx_arrays) {   /* MXFP4 x I8 block scales, address mode: arrays of br pointers */
      if (s->u.gemm.br_type == 1 && xb_rt_ptr_kind(p->a.tertiary) != 1) {
        memcpy(arrays + off, p->a.tertiary, (size_t)r->br * 8); r->a_s = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
      }
      if (s->u.gemm.br_type == 1 && xb_rt_ptr_kind(p->b.tertiary) != 1) {
        memcpy(arrays + off, p->b.tertiary, (size_t)r->br * 8); r->b_s = (char*)plan->d_arrays + off; off += (size_t)r->br * 8;
      }
    }
    if (s->u.gemm.path == P_I8_F32 && p->c.tertiary != NULL) r->scf = *(const float*)p->c.tertiary;
  }
  plan->d_recs = (xb_gemm_rec*)xb_rt_device_malloc((size_t)count * sizeof(xb_gemm_rec));
  if (plan->d_recs == NULL) { free(arrays); free(recs); xb_rt_device_free(plan->d_arrays); free(plan); return NULL; }
  if (arrays_bytes) xb_rt_memcpy(plan->d_arrays, arrays, arrays_bytes);
  xb_rt_memcpy(plan->d_recs, recs, (size_t)count * sizeof(xb_gemm_rec));
  free(arrays); free(recs);
  plan->slot = s; plan->count = count;
  return plan;
}

/* a plan is prepared once and replayed: side operands (xb_gemm_sides) are per-call operands, so such a handle gets no plan */
LIBXSMM_API libxsmm_b200_gemm_plan* libxsmm_b200_gemm_plan_create(libxsmm_gemmfunction kernel,
  const libxsmm_gemm_param* params, long long count)
{
  const xb_slot* s = xb_gemm_slot((const void*)kernel);
  if (s == NULL || xb_gemm_sides(&s->u.gemm) != 0) return NULL;
  return xb_plan_make(s, params, count);
}

LIBXSMM_API int libxsmm_b200_gemm_plan_run(const libxsmm_b200_gemm_plan* plan) {
  xb_gemm_launch L;
  int rc;
  if (plan == NULL) return -1;
  if (plan->pooled) {
    rc = xb_gemm_tc_launch_pooled(&plan->slot->u.gemm, &plan->pool, plan->br, plan->count);
    if (rc == 0 && xb_rt_blocking()) rc = xb_rt_sync();
    return rc;
  }
  memset(&L, 0, sizeof(L));
  L.d = plan->slot->u.gemm; L.count = plan->count; L.recs = plan->d_recs;
  rc = xb_run_gemm_launch(&L);
  if (rc == 0 && xb_rt_blocking()) rc = xb_rt_sync();
  return rc;
}

LIBXSMM_API int libxsmm_b200_gemm_plan_is_pooled(const libxsmm_b200_gemm_plan* plan) { return (plan != NULL && plan->pooled) ? 1 : 0; }

LIBXSMM_API void libxsmm_b200_gemm_plan_destroy(libxsmm_b200_gemm_plan* plan) {
  if (plan == NULL) return;
  xb_rt_device_free(plan->d_recs); xb_rt_device_free(plan->d_arrays); xb_rt_device_free(plan->d_sets); xb_rt_device_free(plan->d_cptrs);
  free(plan);
}

LIBXSMM_API int libxsmm_b200_gemm_batch(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* params, long long count) {
  const xb_slot* s = xb_gemm_slot((const void*)kernel);
  libxsmm_b200_gemm_plan* plan;
  int rc;
  if (s != NULL && xb_batch_refused(&s->u.gemm, 0)) return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
  if (count == 0) return 0;
  plan = xb_plan_make(s, params, count);   /* unlike a plan, one batch call also carries each tile's side operands */
  if (plan == NULL) return -1;
  rc = libxsmm_b200_gemm_plan_run(plan);
  if (rc == 0 && !xb_rt_blocking()) rc = xb_rt_sync();   /* the plan's arrays must outlive the launch */
  libxsmm_b200_gemm_plan_destroy(plan);
  return rc;
}

/* ---- handle invocation switchboard ---------------------------------------------------------------- */
extern void xb_invoke_meltw(const xb_slot* s, const void* param);
extern void xb_invoke_sparse(const xb_slot* s, const libxsmm_gemm_param* param);

void xb_invoke(int slot, const void* param) {
  const xb_slot* s = &g_slots[slot];
  switch (s->kind) {
    case XB_KIND_GEMM: case XB_KIND_GEMM_EXT: xb_invoke_gemm(s, (const libxsmm_gemm_param*)param); break;
    case XB_KIND_TILECFG: break;
    case XB_KIND_MELTW: xb_invoke_meltw(s, param); break;
    case XB_KIND_SP_A_CSR: case XB_KIND_SP_B_CSR: case XB_KIND_SP_B_CSC: case XB_KIND_SP_C_CSC:
    case XB_KIND_BCSC: case XB_KIND_SREG: case XB_KIND_PK_GEMM: case XB_KIND_PK_AC_RM: case XB_KIND_PK_BC_RM:
      xb_invoke_sparse(s, (const libxsmm_gemm_param*)param); break;
    case XB_KIND_MEQN: xb_invoke_meqn(s, param); break;
    default:
      if (libxsmm_verbosity != 0) fprintf(stderr, "LIBXSMM-B200 ERROR: call through a released kernel handle\n");
  }
}

/* ---- introspection ---------------------------------------------------------------------------------- */
extern int xb_user_value_info(const void* value, size_t* size);      /* host_meqn.c: the user registry */
extern int xb_user_value_release(const void* value);
extern void* xb_user_first(const void** key);
extern void* xb_user_next(const void* value, const void** key);

static int xb_public_kind(int kind) {
  return (kind == XB_KIND_MELTW) ? LIBXSMM_KERNEL_KIND_MELTW : ((kind == XB_KIND_MEQN) ? LIBXSMM_KERNEL_KIND_MEQN : LIBXSMM_KERNEL_KIND_MATMUL);
}

LIBXSMM_API int libxsmm_get_kernel_info(const void* kernel, libxsmm_kernel_info* info) {
  const xb_slot* s = xb_slot_of(kernel);
  if (info == NULL) return 1;
  if (s == NULL) {                    /* not a thunk: the value of a user entry? (tests/registry.c:121-126) */
    size_t size = 0;
    if (!xb_user_value_info(kernel, &size)) return 1;
    memset(info, 0, sizeof(*info));
    info->kind = LIBXSMM_KERNEL_KIND_USER; info->code_size = size;
    return 0;
  }
  if (s->kind == XB_KIND_FREE) return 1;
  memset(info, 0, sizeof(*info));
  info->kind = (libxsmm_kernel_kind)xb_public_kind(s->kind);
  info->nflops = s->nflops;
  info->code_size = 16;               /* one trampoline */
  info->is_reference_kernel = 0;
  return 0;
}

LIBXSMM_API int libxsmm_get_mmkernel_info(libxsmm_xmmfunction kernel, libxsmm_mmkernel_info* info) {
  const xb_slot* s = xb_slot_of(kernel.ptr_const);
  if (s == NULL || info == NULL) return 1;
  memset(info, 0, sizeof(*info));
  if (s->kind == XB_KIND_GEMM || s->kind == XB_KIND_GEMM_EXT || s->kind == XB_KIND_TILECFG) {
    const xb_gemm_desc* d = &s->u.gemm;
    info->iprecision = (libxsmm_datatype)d->ta; info->oprecision = (libxsmm_datatype)d->tc;
    info->prefetch = (libxsmm_gemm_prefetch_type)d->prefetch;
    info->lda = (unsigned int)d->lda; info->ldb = (unsigned int)d->ldb; info->ldc = (unsigned int)d->ldc;
    info->m = (unsigned int)d->m; info->n = (unsigned int)d->n; info->k = (unsigned int)d->k; info->flags = (int)d->flags;
    return 0;
  }
  if (s->kind >= XB_KIND_SP_A_CSR) {
    const xb_sparse_desc* d = &s->u.sp;
    info->iprecision = (libxsmm_datatype)d->ta; info->oprecision = (libxsmm_datatype)d->tc;
    info->lda = (unsigned int)d->lda; info->ldb = (unsigned int)d->ldb; info->ldc = (unsigned int)d->ldc;
    info->m = (unsigned int)d->m; info->n = (unsigned int)d->n; info->k = (unsigned int)d->k; info->flags = (int)d->flags;
    return 0;
  }
  return 1;
}

LIBXSMM_API int libxsmm_get_meltwkernel_info(libxsmm_xmeltwfunction kernel, libxsmm_meltwkernel_info* info) {
  const xb_slot* s = xb_slot_of((const void*)kernel.xmeltw);
  if (s == NULL || info == NULL || s->kind != XB_KIND_MELTW) return 1;
  memset(info, 0, sizeof(*info));
  info->ldi = (unsigned int)s->u.meltw.ldi; info->ldo = (unsigned int)s->u.meltw.ldo;
  info->m = (unsigned int)s->u.meltw.m; info->n = (unsigned int)s->u.meltw.n;
  info->datatype = (unsigned int)s->u.meltw.t_in0 | ((unsigned int)s->u.meltw.t_out << 8);
  info->flags = s->u.meltw.flags; info->operation = (unsigned int)s->u.meltw.op_class;
  return 0;
}

LIBXSMM_API int libxsmm_get_registry_info(libxsmm_registry_info* info) {
  if (info == NULL) return 1;
  memset(info, 0, sizeof(*info));
  pthread_mutex_lock(&g_lock);
  info->capacity = XB_REG_CAP / 2; info->size = g_reg_size; info->nbytes = g_reg_size * sizeof(xb_slot);
  pthread_mutex_unlock(&g_lock);
  return 0;
}

LIBXSMM_API int libxsmm_b200_kernel_backend(const void* kernel) {
  const xb_slot* s = xb_slot_of(kernel);
  if (s == NULL) return LIBXSMM_B200_BACKEND_NONE;
  switch (s->kind) {
    case XB_KIND_GEMM: case XB_KIND_GEMM_EXT: return s->u.gemm.backend;
    case XB_KIND_TILECFG: return LIBXSMM_B200_BACKEND_NOOP;
    case XB_KIND_FREE: return LIBXSMM_B200_BACKEND_NONE;
    /* BCSC: which kernel runs also depends on the call-time column count; this is the handle's eligibility (one block-column) */
    case XB_KIND_BCSC: return (xb_bcsc_tc_variant(&s->u.sp, 1) != 0) ? LIBXSMM_B200_BACKEND_TCGEN05 : LIBXSMM_B200_BACKEND_SIMT;
    default: return LIBXSMM_B200_BACKEND_STREAM;
  }
}

LIBXSMM_API int libxsmm_b200_bcsc_variant(const void* kernel, unsigned long long n_block_columns) {
  const xb_slot* s = xb_slot_of(kernel);
  if (s == NULL || s->kind != XB_KIND_BCSC) return -1;
  return xb_bcsc_tc_variant(&s->u.sp, n_block_columns);
}

/* enumeration by kind (reference include/libxsmm.h:105-108): user entries yield their value and key; kernel kinds yield the callable
 * of every REGISTERED handle and the descriptor it is keyed by */
static void* xb_registry_scan(int from, int kind, const void** key) {
  int i; void* result = NULL;
  pthread_mutex_lock(&g_lock);
  for (i = from; i < XB_NTHUNKS; ++i) {
    const xb_slot* s = &g_slots[i];
    if (s->kind != XB_KIND_FREE && s->registered && xb_public_kind(s->kind) == kind) { result = (void*)(uintptr_t)xb_thunk(i); if (key != NULL) *key = &s->u; break; }
  }
  pthread_mutex_unlock(&g_lock);
  return result;
}
LIBXSMM_API void* libxsmm_get_registry_begin(libxsmm_kernel_kind kind, const void** key) {
  LIBXSMM_INIT
  if (kind == LIBXSMM_KERNEL_KIND_USER) return xb_user_first(key);
  return xb_registry_scan(0, (int)kind, key);
}
LIBXSMM_API void* libxsmm_get_registry_next(const void* regentry, const void** key) {
  const xb_slot* s = xb_slot_of(regentry);
  if (regentry == NULL) return NULL;
  if (s == NULL) return xb_user_next(regentry, key);
  return xb_registry_scan((int)(s - g_slots) + 1, xb_public_kind(s->kind), key);
}

LIBXSMM_API void libxsmm_release_kernel(const void* kernel) {
  xb_slot* s = xb_slot_of(kernel);
  if (s == NULL) { (void)xb_user_value_release(kernel); return; }      /* user entries are released through their value */
  if (s->kind == XB_KIND_FREE) return;
  if (s->registered) {   /* reference src/libxsmm_main.c:3916-3921: registered kernels are not released */
    if (libxsmm_verbosity != 0) fprintf(stderr, "LIBXSMM-B200 WARNING: attempt to release a registered kernel\n");
    return;
  }
  pthread_mutex_lock(&g_lock);
  if (s->kind == XB_KIND_MEQN) xb_meqn_release(s->u.sp.work);
  else if (s->kind >= XB_KIND_SP_A_CSR) xb_sparse_release(&s->u.sp);
  memset(s, 0, sizeof(*s));
  pthread_mutex_unlock(&g_lock);
}
