/* libxsmm_b200 -- matrix equations (libxsmm_meqn_*, include/libxsmm.h:149-162) and the user key/value registry
 * (libxsmm_xregister / xdispatch / xrelease, :120-125).
 *
 * An equation is a tree of TPP nodes built in pre-order (push_back_*), exactly the reference's construction
 * (src/libxsmm_matrixeqn.c). The reference then either JITs one fused loop nest or -- its portable path,
 * src/generator_matequation_reference_impl.c:95-227 -- walks an execution plan and runs one mateltwise kernel per node with
 * temporaries typed by the node's own datatype (shape rules: libxsmm_matrixeqn.c:867-925). This file is that second
 * form on the GPU: dispatch infers the shapes, checks that every node is an operation the CUDA mateltwise library has,
 * and returns a handle; a call evaluates the tree bottom-up, one kernel launch per node, temporaries in the
 * stream-ordered scratch arena. GEMM nodes (is_matmul / is_brgemm) are not built: dispatch answers NULL for them.
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"

extern int xb_host_slot_alloc(int kind, unsigned int nflops);
extern xb_slot* xb_host_slot(int i);

#define XB_EQN_MAX 256
#define XB_EQN_NODES 64
enum { EQ_NONE = 0, EQ_ARG, EQ_UNARY, EQ_BINARY, EQ_TERNARY };

typedef struct xb_eqn_node {
  int type, op, dtype; unsigned int flags;
  int pos;                      /* ARG: position in inputs[]; ops: position in ops_args[] */
  int m, n, ld;                 /* result shape (ARG: as declared) */
  int child[3];
  int score;                    /* temporaries the subtree needs; decides which operand subtree runs first (assign_scores) */
} xb_eqn_node;
typedef struct xb_eqn { xb_eqn_node node[XB_EQN_NODES]; int nnodes; int used; } xb_eqn;
typedef struct xb_eqn_plan { xb_eqn eqn; int out_m, out_n, out_ld, out_type; } xb_eqn_plan;

static xb_eqn g_eqn[XB_EQN_MAX];
static int g_neqn = 0;
static pthread_mutex_t g_eqn_lock = PTHREAD_MUTEX_INITIALIZER;

static int arity(int type) { return type == EQ_UNARY ? 1 : (type == EQ_BINARY ? 2 : (type == EQ_TERNARY ? 3 : 0)); }

LIBXSMM_API libxsmm_blasint libxsmm_meqn_create(void) {
  int idx = -1;
  LIBXSMM_INIT
  pthread_mutex_lock(&g_eqn_lock);
  if (g_neqn < XB_EQN_MAX) { idx = g_neqn++; memset(&g_eqn[idx], 0, sizeof(g_eqn[idx])); g_eqn[idx].used = 1; }
  pthread_mutex_unlock(&g_eqn_lock);
  return idx;
}
LIBXSMM_API libxsmm_meqn_arg_shape libxsmm_create_meqn_arg_shape(const libxsmm_blasint m, const libxsmm_blasint n, const libxsmm_blasint ld, const libxsmm_datatype type) {
  libxsmm_meqn_arg_shape r; r.m = m; r.n = n; r.ld = ld; r.type = type; return r;
}
LIBXSMM_API libxsmm_matrix_arg_attributes libxsmm_create_matrix_arg_attributes(const libxsmm_matrix_arg_type type, const libxsmm_matrix_arg_set_type set_type,
  const libxsmm_blasint set_cardinality_hint, const libxsmm_blasint set_stride_hint) {
  libxsmm_matrix_arg_attributes r; r.type = type; r.set_type = set_type; r.set_cardinality_hint = set_cardinality_hint; r.set_stride_hint = set_stride_hint; return r;
}
LIBXSMM_API libxsmm_meqn_arg_metadata libxsmm_create_meqn_arg_metadata(const libxsmm_blasint eqn_idx, const libxsmm_blasint in_arg_pos) {
  libxsmm_meqn_arg_metadata r; r.eqn_idx = eqn_idx; r.in_arg_pos = in_arg_pos; return r;
}
LIBXSMM_API libxsmm_meqn_op_metadata libxsmm_create_meqn_op_metadata(const libxsmm_blasint eqn_idx, const libxsmm_blasint op_arg_pos) {
  libxsmm_meqn_op_metadata r; r.eqn_idx = eqn_idx; r.op_arg_pos = op_arg_pos; return r;
}

/* first free child slot in pre-order; *parent = -1: the tree is empty (the new node becomes the root); returns 0 if the tree is complete */
static int find_slot(const xb_eqn* e, int at, int* parent, int* which) {
  int c;
  if (e->nnodes == 0) { *parent = -1; *which = 0; return 1; }
  for (c = 0; c < arity(e->node[at].type); ++c) {
    if (e->node[at].child[c] < 0) { *parent = at; *which = c; return 1; }
    if (find_slot(e, e->node[at].child[c], parent, which)) return 1;
  }
  return 0;
}
static int push_node(int eqn_idx, const xb_eqn_node* proto) {
  xb_eqn* e; int parent, which, rc = 1;
  if (eqn_idx < 0 || eqn_idx >= g_neqn) return 1;
  pthread_mutex_lock(&g_eqn_lock);
  e = &g_eqn[eqn_idx];
  if (e->nnodes < XB_EQN_NODES && find_slot(e, 0, &parent, &which)) {
    const int id = e->nnodes++;
    e->node[id] = *proto; e->node[id].child[0] = e->node[id].child[1] = e->node[id].child[2] = -1;
    if (parent >= 0) e->node[parent].child[which] = id;
    rc = 0;
  }
  pthread_mutex_unlock(&g_eqn_lock);
  return rc;
}
LIBXSMM_API int libxsmm_meqn_push_back_arg(const libxsmm_meqn_arg_metadata arg_metadata, const libxsmm_meqn_arg_shape arg_shape, libxsmm_matrix_arg_attributes arg_attr) {
  xb_eqn_node nd; memset(&nd, 0, sizeof(nd));
  if (arg_attr.type != LIBXSMM_MATRIX_ARG_TYPE_SINGULAR) return 1;          /* argument sets only feed BRGEMM nodes */
  nd.type = EQ_ARG; nd.pos = arg_metadata.in_arg_pos; nd.m = arg_shape.m; nd.n = arg_shape.n; nd.ld = arg_shape.ld; nd.dtype = (int)arg_shape.type;
  return push_node(arg_metadata.eqn_idx, &nd);
}
LIBXSMM_API int libxsmm_meqn_push_back_unary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_unary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags) {
  xb_eqn_node nd; memset(&nd, 0, sizeof(nd));
  nd.type = EQ_UNARY; nd.op = (int)type; nd.dtype = (int)dtype; nd.flags = flags; nd.pos = op_metadata.op_arg_pos;
  return push_node(op_metadata.eqn_idx, &nd);
}
LIBXSMM_API int libxsmm_meqn_push_back_binary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_binary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags) {
  xb_eqn_node nd; memset(&nd, 0, sizeof(nd));
  nd.type = EQ_BINARY; nd.op = (int)type; nd.dtype = (int)dtype; nd.flags = flags; nd.pos = op_metadata.op_arg_pos;
  return push_node(op_metadata.eqn_idx, &nd);
}
LIBXSMM_API int libxsmm_meqn_push_back_ternary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_ternary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags) {
  xb_eqn_node nd; memset(&nd, 0, sizeof(nd));
  nd.type = EQ_TERNARY; nd.op = (int)type; nd.dtype = (int)dtype; nd.flags = flags; nd.pos = op_metadata.op_arg_pos;
  return push_node(op_metadata.eqn_idx, &nd);
}

static void print_tree(const xb_eqn* e, int at, int depth, int rpn) {
  int c; const xb_eqn_node* nd = &e->node[at];
  static const char* names[] = { "?", "ARG", "UNARY", "BINARY", "TERNARY" };
  if (rpn) for (c = 0; c < arity(nd->type); ++c) if (nd->child[c] >= 0) print_tree(e, nd->child[c], depth + 1, rpn);
  if (nd->type == EQ_ARG) printf("%*sARG in_pos=%d %dx%d ld=%d dtype=%d\n", rpn ? 0 : 2 * depth, "", nd->pos, nd->m, nd->n, nd->ld, nd->dtype);
  else printf("%*s%s op=%d flags=%u dtype=%d\n", rpn ? 0 : 2 * depth, "", names[nd->type], nd->op, nd->flags, nd->dtype);
  if (!rpn) for (c = 0; c < arity(nd->type); ++c) if (nd->child[c] >= 0) print_tree(e, nd->child[c], depth + 1, rpn);
}
LIBXSMM_API void libxsmm_meqn_tree_print(const libxsmm_blasint idx) { if (idx >= 0 && idx < g_neqn && g_eqn[idx].nnodes > 0) print_tree(&g_eqn[idx], 0, 0, 0); }
LIBXSMM_API void libxsmm_meqn_rpn_print(const libxsmm_blasint idx) { if (idx >= 0 && idx < g_neqn && g_eqn[idx].nnodes > 0) print_tree(&g_eqn[idx], 0, 0, 1); }

/* ---- shapes (src/libxsmm_matrixeqn.c:867-925) and per-node kernel descriptors ----------------------------------------- */
static int is_reduce(int op) {
  return op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD
      || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX;
}
static int infer(xb_eqn* e, int at) {
  xb_eqn_node* nd = &e->node[at]; int c;
  for (c = 0; c < arity(nd->type); ++c) { if (nd->child[c] < 0 || infer(e, nd->child[c]) != 0) return 1; }
  if (nd->type == EQ_UNARY) {
    const xb_eqn_node* le = &e->node[nd->child[0]];
    if (is_reduce(nd->op)) {
      if (nd->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) { nd->m = le->n; nd->n = 1; nd->ld = le->n; }
      else if (nd->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_COLS) { nd->m = le->m; nd->n = 1; nd->ld = le->m; }
      else return 1;
    } else if (nd->op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD) { nd->m = nd->n = nd->ld = 1; }
    else if (nd->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT) { nd->m = le->n; nd->n = le->m; nd->ld = le->n; }
    else { nd->m = le->m; nd->n = le->n; nd->ld = le->m; }
  } else if (nd->type == EQ_BINARY) {
    const xb_eqn_node *le = &e->node[nd->child[0]], *ri = &e->node[nd->child[1]];
    if (nd->op == LIBXSMM_MELTW_TYPE_BINARY_MATMUL || (nd->op >= LIBXSMM_MELTW_TYPE_BINARY_BRGEMM && nd->op <= LIBXSMM_MELTW_TYPE_BINARY_MATMUL_A_VNNI_TRANS_B_TRANS)) return 1;   /* GEMM nodes: not built */
    if (nd->op == LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD) { nd->m = nd->n = nd->ld = 1; }
    else { nd->m = LIBXSMM_MAX(le->m, ri->m); nd->n = LIBXSMM_MAX(le->n, ri->n); nd->ld = nd->m; }
  } else if (nd->type == EQ_TERNARY) {
    const xb_eqn_node *le = &e->node[nd->child[0]], *ri = &e->node[nd->child[1]], *r2 = &e->node[nd->child[2]];
    if (nd->op != LIBXSMM_MELTW_TYPE_TERNARY_SELECT && nd->op != LIBXSMM_MELTW_TYPE_TERNARY_MULADD && nd->op != LIBXSMM_MELTW_TYPE_TERNARY_NMULADD) return 1;
    nd->m = LIBXSMM_MAX(r2->m, LIBXSMM_MAX(le->m, ri->m)); nd->n = LIBXSMM_MAX(r2->n, LIBXSMM_MAX(le->n, ri->n)); nd->ld = nd->m;
  }
  return 0;
}
/* the mateltwise descriptor the reference builds for this node (generator_matequation_reference_impl.c:107-206) */
static void node_desc(const xb_eqn* e, int at, xb_meltw_desc* d) {
  const xb_eqn_node* nd = &e->node[at];
  const xb_eqn_node* le = &e->node[nd->child[0]];
  memset(d, 0, sizeof(*d));
  d->op = nd->op; d->flags = nd->flags; d->t_in0 = le->dtype; d->t_out = nd->dtype; d->t_comp = nd->dtype;
  d->t_in1 = d->t_in2 = LIBXSMM_DATATYPE_UNSUPPORTED;
  d->ldi = le->ld; d->ldo = nd->ld; d->m = nd->m; d->n = nd->n;
  if (nd->type == EQ_UNARY) {
    d->op_class = LIBXSMM_MELTW_OPERATION_UNARY;
    if (is_reduce(nd->op) || nd->op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD || nd->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT) { d->m = le->m; d->n = le->n; }
    if (nd->op == LIBXSMM_MELTW_TYPE_UNARY_IDENTITY && le->dtype != nd->dtype) d->t_comp = LIBXSMM_DATATYPE_F32;
  } else if (nd->type == EQ_BINARY) {
    const xb_eqn_node* ri = &e->node[nd->child[1]];
    d->op_class = LIBXSMM_MELTW_OPERATION_BINARY; d->t_in1 = ri->dtype; d->ldi2 = ri->ld;
    if (nd->op == LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD) { d->m = LIBXSMM_MAX(le->m, ri->m); d->n = LIBXSMM_MAX(le->n, ri->n); }
  } else {
    const xb_eqn_node *ri = &e->node[nd->child[1]], *r2 = &e->node[nd->child[2]];
    d->op_class = LIBXSMM_MELTW_OPERATION_TERNARY; d->t_in1 = ri->dtype; d->ldi2 = ri->ld; d->ldi3 = r2->ld;
    d->t_in2 = (nd->op == LIBXSMM_MELTW_TYPE_TERNARY_SELECT) ? LIBXSMM_DATATYPE_IMPLICIT : r2->dtype;
  }
}
/* Order of evaluation. The reference runs, below every node, the operand subtree that needs MORE temporaries first (ties: left to
 * right) -- a Sethi-Ullman numbering with its own twists (src/libxsmm_matrixeqn.c:323-400 scores, :745-790 visiting order). The order is
 * observable: a DUMP node writes caller memory that another branch may read as an argument (equation_softmax.c,
 * equation_bf16_x3_split_f32.c), so the numbering is restated here: an argument needs 0; a node over arguments only needs 1; a unary
 * node inherits its operand's count when it may overwrite the operand's temporary and needs at least 2 otherwise; a binary node needs
 * one more than two equally demanding operands, else the larger count, and at least 3 when it may not overwrite; a ternary node needs
 * the largest operand count and at least 4 (3 when it reuses its third operand as output). "May overwrite" fails for IDENTITY, for
 * layout transforms, for GEMM nodes and whenever an 8/16-bit float operand is widened to F32/F64 (:196-223). */
static int is_narrow_float(int t) { return t == LIBXSMM_DATATYPE_BF16 || t == LIBXSMM_DATATYPE_F16 || t == LIBXSMM_DATATYPE_BF8 || t == LIBXSMM_DATATYPE_HF8; }
static int is_wide_float(int t) { return t == LIBXSMM_DATATYPE_F32 || t == LIBXSMM_DATATYPE_F64; }
static int is_layout_transform(int op) {
#define XB_IS_TRANSFORM(NAME, VALUE) if (op == (VALUE)) return 0 == strncmp(#NAME, "TRANSFORM_", 10);
  LIBXSMM_B200_UNARY_TYPES(XB_IS_TRANSFORM)
#undef XB_IS_TRANSFORM
  return 0;
}
static void assign_scores(xb_eqn* e, int at) {
  xb_eqn_node* nd = &e->node[at]; int c, all_args = 1, top = 0, widened = 0;
  if (nd->type == EQ_ARG) { nd->score = 0; return; }
  for (c = 0; c < arity(nd->type); ++c) {
    const xb_eqn_node* ch;
    assign_scores(e, nd->child[c]);
    ch = &e->node[nd->child[c]];
    if (ch->type != EQ_ARG) all_args = 0;
    if (ch->score > top) top = ch->score;
    if (is_narrow_float(ch->dtype) && is_wide_float(nd->dtype)) widened = 1;
  }
  if (all_args) { nd->score = 1; return; }
  if (nd->type == EQ_UNARY) {
    const int in_place = !(nd->op == LIBXSMM_MELTW_TYPE_UNARY_IDENTITY || is_layout_transform(nd->op) || widened);
    nd->score = in_place ? top : LIBXSMM_MAX(2, top);
  } else if (nd->type == EQ_BINARY) {
    const int l = e->node[nd->child[0]].score, r = e->node[nd->child[1]].score, need = (l == r) ? l + 1 : top;
    const int in_place = !(nd->op == LIBXSMM_MELTW_TYPE_BINARY_MATMUL || nd->op == LIBXSMM_MELTW_TYPE_BINARY_BRGEMM || widened);
    nd->score = in_place ? need : LIBXSMM_MAX(3, need);
  } else {
    nd->score = LIBXSMM_MAX((nd->flags & LIBXSMM_MELTW_FLAG_TERNARY_REUSE_IN_2_AS_OUT) ? 3 : 4, top);
  }
}

/* the side operands of a node's kernel (xb_meltw_sides); an argument has none */
static int node_sides(const xb_eqn* e, int at) {
  xb_meltw_desc d;
  if (e->node[at].type == EQ_ARG) return 0;
  node_desc(e, at, &d);
  return xb_meltw_sides(&d);
}

static int check_nodes(const xb_eqn* e, int at) {
  const xb_eqn_node* nd = &e->node[at]; int c, unwired; xb_meltw_desc d;
  if (nd->type == EQ_ARG) return 0;
  for (c = 0; c < arity(nd->type); ++c) if (check_nodes(e, nd->child[c]) != 0) return 1;
  node_desc(e, at, &d);
  /* declined rather than mis-evaluated: nodes without a storage type (IMPLICIT: zip / unzip trees) and nodes with side operands this
   * evaluator does not wire (samples/equation/equation_splitSGD.c, equation_gather_*.c, equation_bf16_x3_split_f32.c). It wires the
   * bit mask of a relu at the head, the copy of a DUMP and an alpha from ops_args. */
  if (libxsmm_typesize((libxsmm_datatype)nd->dtype) == 0 || xb_meltw_family(&d) == XB_FAM_NONE) return 1;
  unwired = xb_meltw_sides(&d) & ~(XB_MSIDE_MASK_OUT | XB_MSIDE_COPY_OUT | XB_MSIDE_ALPHA);
  /* kept as they were (follow-ups): an argop reduction is accepted and its indices are not recorded; a unary node with STOCHASTIC_ROUND
   * is declined whatever its op; a binary or ternary one is accepted and its generator state is not wired */
  unwired &= ~XB_MSIDE_ARGOP;
  if (nd->type != EQ_UNARY) unwired &= ~XB_MSIDE_STATE;
  else if (nd->flags & LIBXSMM_MELTW_FLAG_UNARY_STOCHASTIC_ROUND) return 1;
  /* a relu's bit mask has one destination, output.secondary: only the head may produce it (reference :39-56) */
  return (unwired != 0 || (at != 0 && (xb_meltw_sides(&d) & XB_MSIDE_MASK_OUT))) ? 1 : 0;
}

LIBXSMM_API libxsmm_meqn_function libxsmm_dispatch_meqn(const libxsmm_blasint idx, const libxsmm_meqn_arg_shape out_shape) {
  xb_eqn_plan* plan; int slot, parent, which; xb_slot* s; xb_eqn_node* root;
  LIBXSMM_INIT
  if (idx < 0 || idx >= g_neqn || g_eqn[idx].nnodes == 0 || !xb_rt_have_gpu()) return NULL;
  plan = (xb_eqn_plan*)calloc(1, sizeof(*plan));
  if (plan == NULL) return NULL;
  pthread_mutex_lock(&g_eqn_lock); plan->eqn = g_eqn[idx]; pthread_mutex_unlock(&g_eqn_lock);
  if (find_slot(&plan->eqn, 0, &parent, &which) /* incomplete */ || plan->eqn.node[0].type == EQ_ARG || infer(&plan->eqn, 0) != 0) { free(plan); return NULL; }
  root = &plan->eqn.node[0];
  root->ld = out_shape.ld; root->dtype = (int)out_shape.type;       /* the head writes the caller's output */
  if (out_shape.m != root->m || out_shape.n != root->n) {            /* reductions: the caller passes the result extents too */
    if ((long long)out_shape.m * out_shape.n != (long long)root->m * root->n) { free(plan); return NULL; }
  }
  if (check_nodes(&plan->eqn, 0) != 0) { free(plan); return NULL; }
  assign_scores(&plan->eqn, 0);
  plan->out_m = root->m; plan->out_n = root->n; plan->out_ld = out_shape.ld; plan->out_type = (int)out_shape.type;
  slot = xb_host_slot_alloc(XB_KIND_MEQN, 0);
  if (slot < 0) { free(plan); return NULL; }
  s = xb_host_slot(slot);
  memset(&s->u, 0, sizeof(s->u));
  s->u.sp.kind = XB_KIND_MEQN; s->u.sp.work = plan;
  return (libxsmm_meqn_function)xb_thunk(slot);
}
void xb_meqn_release(void* work) { free(work); }

/* ---- evaluation --------------------------------------------------------------------------------------------------- */
typedef struct xb_eval {
  const xb_eqn* e; const libxsmm_meqn_param* p; void* out_dev; int failed;
  struct { void* host; void* dev; size_t bytes; } back[4]; int nback;   /* secondary outputs staged for host callers */
} xb_eval;

static size_t span(const xb_eqn_node* nd) { return ((size_t)(nd->n - 1) * nd->ld + nd->m) * libxsmm_typesize((libxsmm_datatype)nd->dtype); }

/* a secondary output (relu bit mask, dump copy): device pointers pass through, host memory is staged in and copied back at the end */
static void* eval_aux_out(xb_eval* ev, void* user, size_t bytes) {
  void* d;
  if (user == NULL || bytes == 0) { ev->failed = 1; return NULL; }
  if (xb_rt_ptr_kind(user) != 0) return user;
  if (ev->nback >= (int)(sizeof(ev->back) / sizeof(ev->back[0]))) { ev->failed = 1; return NULL; }
  d = xb_rt_scratch(bytes);
  if (d == NULL) { ev->failed = 1; return NULL; }
  xb_rt_upload(d, user, bytes);
  ev->back[ev->nback].host = user; ev->back[ev->nback].dev = d; ev->back[ev->nback].bytes = bytes; ev->nback++;
  return d;
}
static int has_bitmask_out(const xb_eqn* e, int at) { return (node_sides(e, at) & XB_MSIDE_MASK_OUT) != 0; }
/* the alpha of a node that takes one (xb_meltw_sides: ALPHA), from its ops_args slot of call 0; 1 otherwise */
static float node_alpha(const xb_eqn* e, int at, const libxsmm_meqn_param* p) {
  const xb_eqn_node* nd = &e->node[at];
  if ((node_sides(e, at) & XB_MSIDE_ALPHA) == 0 || p->ops_args == NULL || nd->pos < 0 || p->ops_args[nd->pos].primary == NULL) return 1.0f;
  return xb_meltw_scalar(p->ops_args[nd->pos].primary);
}

static const void* eval_node(xb_eval* ev, int at, int is_root) {
  const xb_eqn_node* nd = &ev->e->node[at];
  if (nd->type == EQ_ARG) {
    const void* hp = ev->p->inputs[nd->pos].primary;
    if (hp == NULL) { ev->failed = 1; return NULL; }
    if (xb_rt_ptr_kind(hp) != 0) return hp;
    { int i;   /* host memory an earlier node of this evaluation wrote as its secondary output (softmax: DUMP -> tmp -> operand) */
      for (i = 0; i < ev->nback; ++i) if (ev->back[i].host == hp && ev->back[i].bytes >= span(nd)) return ev->back[i].dev; }
    { void* d = xb_rt_scratch(span(nd)); if (d == NULL) { ev->failed = 1; return NULL; } xb_rt_upload(d, hp, span(nd)); return d; }
  } else {
    xb_meltw_desc d; xb_meltw_args a; void* out;
    const void* in[3] = { NULL, NULL, NULL }; int c, k, order[3] = { 0, 1, 2 };
    memset(&a, 0, sizeof(a));
    /* the more demanding operand subtree first, ties left to right (assign_scores); plain arguments score 0, so they are read last:
     * the reference reads an argument when the consuming node executes, after every operation below that node has run (and possibly
     * written the argument's memory through a DUMP) */
    for (c = 1; c < arity(nd->type); ++c) for (k = c; k > 0 && ev->e->node[nd->child[order[k]]].score > ev->e->node[nd->child[order[k - 1]]].score; --k) {
      const int t = order[k]; order[k] = order[k - 1]; order[k - 1] = t;
    }
    for (c = 0; c < arity(nd->type); ++c) in[order[c]] = eval_node(ev, nd->child[order[c]], 0);
    a.in0 = in[0]; a.in1 = in[1]; a.in2 = in[2];
    if (ev->failed) return NULL;
    out = is_root ? ev->out_dev : xb_rt_scratch(span(nd) ? span(nd) : 16);
    if (out == NULL) { ev->failed = 1; return NULL; }
    node_desc(ev->e, at, &d);
    a.out = out; a.alpha = node_alpha(ev->e, at, ev->p);
    /* secondary outputs as the reference wires them (generator_matequation_reference_impl.c:39-61): the bit mask of a relu at
     * the head goes to output.secondary, a DUMP node copies its value to its ops_args slot */
    if (has_bitmask_out(ev->e, at)) {
      if (!is_root) { ev->failed = 1; return NULL; }
      a.out_aux = eval_aux_out(ev, ev->p->output.secondary, xb_meltw_mask_bytes(d.ldo, d.n));
    } else if (nd->type == EQ_UNARY && nd->op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) {
      a.out_aux = eval_aux_out(ev, (ev->p->ops_args != NULL && nd->pos >= 0) ? ev->p->ops_args[nd->pos].primary : NULL, span(nd));
    }
    if (ev->failed) return NULL;
    if (0 != xb_meltw_launch(&d, &a)) ev->failed = 1;
    return out;
  }
}

void xb_invoke_meqn(const xb_slot* s, const void* param) {
  const xb_eqn_plan* plan = (const xb_eqn_plan*)s->u.sp.work;
  const libxsmm_meqn_param* p = (const libxsmm_meqn_param*)param;
  xb_eval ev; void* host_out = NULL; size_t out_bytes; int i;
  if (plan == NULL || p == NULL || p->output.primary == NULL) return;
  out_bytes = ((size_t)(plan->out_n - 1) * plan->out_ld + plan->out_m) * libxsmm_typesize((libxsmm_datatype)plan->out_type);
  ev.e = &plan->eqn; ev.p = p; ev.failed = 0; ev.nback = 0; ev.out_dev = p->output.primary;
  if (xb_rt_ptr_kind(p->output.primary) == 0) {            /* host output: staged in and out (partial writes keep the padding) */
    host_out = p->output.primary; ev.out_dev = xb_rt_scratch(out_bytes);
    if (ev.out_dev == NULL) { xb_rt_note_error(2, "meqn: out of scratch"); return; }
    xb_rt_upload(ev.out_dev, host_out, out_bytes);
  }
  (void)eval_node(&ev, 0, 1);
  if (ev.failed) { xb_rt_note_error(2, "meqn: evaluation failed"); xb_rt_scratch_reset(); return; }
  if (host_out != NULL) xb_rt_memcpy_async(host_out, ev.out_dev, out_bytes);
  for (i = 0; i < ev.nback; ++i) xb_rt_memcpy_async(ev.back[i].host, ev.back[i].dev, ev.back[i].bytes);
  xb_rt_sync(); xb_rt_scratch_reset();
}

/* ---- strided batch: the tree evaluated once for `count` calls, every node one launch over all of them ------------------------
 * Call t reads inputs[i] + t*input_strides[i] and writes output.primary + t*output_stride (the relu bit mask of the head:
 * output.secondary + t*output_aux_stride, a DUMP: ops_args[pos].primary + t*ops_strides[pos]). A temporary holds its node's value for
 * every call of a chunk at 256-byte aligned strides; when all temporaries of a batch would exceed XB_MEQN_BATCH_SCRATCH_BYTES the
 * calls run in chunks, each one launch per node, then a sync and a scratch reset. */
#define XB_MEQN_BATCH_SCRATCH_BYTES (64ll << 20)

typedef struct xb_beval {
  const xb_eqn* e; const libxsmm_meqn_param* p; const long long* in_s; const long long* ops_s; long long out_s, aux_s, t0, cnt; int failed, rc;
  char* pool; size_t used;      /* the chunk's temporaries: one scratch block, carved in visiting order */
} xb_beval;

static long long tmp_stride(const xb_eqn_node* nd) { return (long long)LIBXSMM_UP(span(nd) ? span(nd) : 16, 256); }
static int is_dump(const xb_eqn_node* nd) { return nd->type == EQ_UNARY && nd->op == LIBXSMM_MELTW_TYPE_UNARY_DUMP; }

static const void* beval_node(xb_beval* ev, int at, int is_root, long long* stride) {
  const xb_eqn_node* nd = &ev->e->node[at];
  if (nd->type == EQ_ARG) {
    /* an argument that a DUMP of this evaluation writes is the DUMP's strided buffer (the entry point checked the strides agree) */
    *stride = ev->in_s[nd->pos];
    return (const char*)ev->p->inputs[nd->pos].primary + ev->t0 * *stride;
  } else {
    xb_meltw_desc d; xb_meltw_args a; char* out;
    const void* in[3] = { NULL, NULL, NULL }; long long s[3] = { 0, 0, 0 }; int c, k, order[3] = { 0, 1, 2 };
    memset(&a, 0, sizeof(a));
    for (c = 1; c < arity(nd->type); ++c) for (k = c; k > 0 && ev->e->node[nd->child[order[k]]].score > ev->e->node[nd->child[order[k - 1]]].score; --k) {
      const int t = order[k]; order[k] = order[k - 1]; order[k - 1] = t;
    }
    for (c = 0; c < arity(nd->type); ++c) in[order[c]] = beval_node(ev, nd->child[order[c]], 0, &s[order[c]]);
    if (ev->failed) return NULL;
    *stride = is_root ? ev->out_s : tmp_stride(nd);
    if (is_root) out = (char*)ev->p->output.primary + ev->t0 * ev->out_s;
    else { out = ev->pool + ev->used; ev->used += (size_t)(ev->cnt * *stride); }
    node_desc(ev->e, at, &d);
    a.in0 = in[0]; a.in1 = in[1]; a.in2 = in[2]; a.s_in0 = s[0]; a.s_in1 = s[1]; a.s_in2 = s[2];
    a.out = out; a.s_out = *stride; a.alpha = node_alpha(ev->e, at, ev->p); a.count = ev->cnt;
    if (has_bitmask_out(ev->e, at)) { a.out_aux = (char*)ev->p->output.secondary + ev->t0 * ev->aux_s; a.s_out_aux = ev->aux_s; }
    else if (is_dump(nd)) { a.out_aux = (char*)ev->p->ops_args[nd->pos].primary + ev->t0 * ev->ops_s[nd->pos]; a.s_out_aux = ev->ops_s[nd->pos]; }
    if (0 != (ev->rc = xb_meltw_launch(&d, &a))) ev->failed = 1;
    return out;
  }
}

LIBXSMM_API int libxsmm_b200_meqn_batch_strided(libxsmm_meqn_function kernel, const libxsmm_meqn_param* param,
  const long long* input_strides, long long output_stride, long long output_aux_stride, const long long* ops_strides, long long count)
{
  const xb_slot* s = xb_slot_of((const void*)kernel);
  const xb_eqn_plan* plan; const xb_eqn* e;
  long long per_tile = 0, chunk, t0;
  int i, rc = 0;
  if (s == NULL || s->kind != XB_KIND_MEQN || param == NULL || param->output.primary == NULL || count < 0) return -1;
  plan = (const xb_eqn_plan*)s->u.sp.work; e = &plan->eqn;
  for (i = 0; i < e->nnodes; ++i) {
    const xb_eqn_node* nd = &e->node[i]; xb_meltw_desc d;
    if (nd->type == EQ_ARG) continue;
    node_desc(e, i, &d);
    if (!xb_meltw_batchable(&d)) return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
  }
  if (output_stride < 0 || output_aux_stride < 0) return -1;
  for (i = 0; i < e->nnodes; ++i) {
    const xb_eqn_node* nd = &e->node[i];
    if (nd->type == EQ_ARG && (input_strides == NULL || param->inputs == NULL || input_strides[nd->pos] < 0 || param->inputs[nd->pos].primary == NULL)) return -1;
    if (is_dump(nd) && (nd->pos < 0 || ops_strides == NULL || param->ops_args == NULL || ops_strides[nd->pos] < 0)) return -1;
    if (has_bitmask_out(e, i) && param->output.secondary == NULL) return -1;
    if (is_dump(nd) && param->ops_args[nd->pos].primary == NULL) return -1;
  }
  /* an argument that a DUMP writes is read through the DUMP's buffer: both strides must describe the same tiles */
  for (i = 0; i < e->nnodes; ++i) if (is_dump(&e->node[i])) {
    const int dp = e->node[i].pos; int j;
    for (j = 0; j < e->nnodes; ++j) {
      const xb_eqn_node* x = &e->node[j];
      if (x->type == EQ_ARG && param->inputs[x->pos].primary == param->ops_args[dp].primary && input_strides[x->pos] != ops_strides[dp]) return -1;
    }
  }
  if (count == 0) return 0;
  if (count > 1) {                      /* calls must not overlap in what they write */
    const size_t out_bytes = ((size_t)(plan->out_n - 1) * plan->out_ld + plan->out_m) * libxsmm_typesize((libxsmm_datatype)plan->out_type);
    if (output_stride < (long long)out_bytes) return -1;
    for (i = 0; i < e->nnodes; ++i) {
      const xb_eqn_node* nd = &e->node[i];
      if (has_bitmask_out(e, i) && output_aux_stride < (long long)xb_meltw_mask_bytes(nd->ld, nd->n)) return -1;
      if (is_dump(nd) && ops_strides[nd->pos] < (long long)span(nd)) return -1;
    }
  }
  /* device-accessible operands only: there is no staging path */
  if (xb_rt_ptr_kind(param->output.primary) == 0) return -4;
  for (i = 0; i < e->nnodes; ++i) {
    const xb_eqn_node* nd = &e->node[i];
    if (nd->type == EQ_ARG && xb_rt_ptr_kind(param->inputs[nd->pos].primary) == 0) return -4;
    if (is_dump(nd) && xb_rt_ptr_kind(param->ops_args[nd->pos].primary) == 0) return -4;
    if (has_bitmask_out(e, i) && xb_rt_ptr_kind(param->output.secondary) == 0) return -4;
    if (nd->type != EQ_ARG && i != 0) per_tile += tmp_stride(nd);
  }
  chunk = (per_tile > 0 && per_tile < XB_MEQN_BATCH_SCRATCH_BYTES) ? XB_MEQN_BATCH_SCRATCH_BYTES / per_tile : (per_tile > 0 ? 1 : count);
  for (t0 = 0; t0 < count && rc == 0; t0 += chunk) {
    xb_beval ev; long long st; int rs;
    memset(&ev, 0, sizeof(ev));
    ev.e = e; ev.p = param; ev.in_s = input_strides; ev.ops_s = ops_strides; ev.out_s = output_stride; ev.aux_s = output_aux_stride;
    ev.t0 = t0; ev.cnt = (count - t0 < chunk) ? count - t0 : chunk;
    ev.pool = (per_tile > 0) ? (char*)xb_rt_scratch((size_t)(per_tile * ev.cnt)) : NULL;
    if (per_tile > 0 && ev.pool == NULL) { xb_rt_note_error(2, "meqn batch: out of scratch"); return 2; }
    (void)beval_node(&ev, 0, 1, &st);
    rc = ev.failed ? (ev.rc != 0 ? ev.rc : 2) : 0;
    if (ev.failed) xb_rt_note_error(rc, "meqn batch: evaluation failed");
    rs = xb_rt_sync();
    if (rc == 0) rc = rs;
    xb_rt_scratch_reset();
  }
  return rc;
}

/* ---- user registry: libxsmm_xregister / xdispatch / xrelease (src/libxsmm_main.c:3010-3120) --------------------------------
 * binary keys of up to LIBXSMM_DESCRIPTOR_MAXSIZE bytes; the value is copied and owned here. A released entry stays in the list as
 * a tombstone (its memory too) until the same key is registered again: tests/registry.c:133-137 walks the registry releasing each
 * entry and then asks for the successor OF THE ENTRY IT JUST RELEASED, so the address has to stay unique and findable. */
typedef struct xb_user_entry { unsigned char key[LIBXSMM_DESCRIPTOR_MAXSIZE]; size_t key_size; void* value; size_t value_size, capacity; int dead; struct xb_user_entry* next; } xb_user_entry;
static xb_user_entry* g_user = NULL;
static pthread_mutex_t g_user_lock = PTHREAD_MUTEX_INITIALIZER;

static xb_user_entry* user_find(const void* key, size_t key_size) {
  xb_user_entry* e;
  for (e = g_user; e != NULL; e = e->next) if (e->key_size == key_size && 0 == memcmp(e->key, key, key_size)) return e;
  return NULL;
}
static xb_user_entry* user_of_value(const void* value) {
  xb_user_entry* e;
  for (e = g_user; e != NULL; e = e->next) if (e->value == value) return e;
  return NULL;
}
LIBXSMM_API void* libxsmm_xregister(const void* key, size_t key_size, size_t value_size, const void* value_init) {
  xb_user_entry* e; void* result = NULL;
  LIBXSMM_INIT
  if (key == NULL || key_size == 0 || key_size > LIBXSMM_DESCRIPTOR_MAXSIZE || value_size == 0) return NULL;
  pthread_mutex_lock(&g_user_lock);
  e = user_find(key, key_size);
  if (e != NULL && e->dead == 0) {       /* an existing key keeps its value unless the new one fits and an initial value is given */
    if (value_size <= e->value_size) { if (value_init != NULL) memcpy(e->value, value_init, value_size); result = e->value; }
  } else if (e != NULL) {                /* a released key comes back, with room for the new payload */
    if (value_size > e->capacity) { void* v = realloc(e->value, value_size); if (v != NULL) { e->value = v; e->capacity = value_size; } }
    if (value_size <= e->capacity) {
      if (value_init != NULL) memcpy(e->value, value_init, value_size); else memset(e->value, 0, value_size);
      e->value_size = value_size; e->dead = 0; result = e->value;
    }
  } else {
    e = (xb_user_entry*)calloc(1, sizeof(*e));
    if (e != NULL) {
      e->value = malloc(value_size);
      if (e->value != NULL) {
        memcpy(e->key, key, key_size); e->key_size = key_size; e->value_size = e->capacity = value_size;
        if (value_init != NULL) memcpy(e->value, value_init, value_size); else memset(e->value, 0, value_size);
        e->next = g_user; g_user = e; result = e->value;
      } else free(e);
    }
  }
  pthread_mutex_unlock(&g_user_lock);
  return result;
}
LIBXSMM_API void* libxsmm_xdispatch(const void* key, size_t key_size) {
  xb_user_entry* e; void* result = NULL;
  if (key == NULL || key_size == 0 || key_size > LIBXSMM_DESCRIPTOR_MAXSIZE) return NULL;
  pthread_mutex_lock(&g_user_lock);
  e = user_find(key, key_size); if (e != NULL && e->dead == 0) result = e->value;
  pthread_mutex_unlock(&g_user_lock);
  return result;
}
LIBXSMM_API void libxsmm_xrelease(const void* key, size_t key_size) {
  xb_user_entry* e;
  if (key == NULL || key_size == 0) return;
  pthread_mutex_lock(&g_user_lock);
  e = user_find(key, key_size); if (e != NULL) e->dead = 1;
  pthread_mutex_unlock(&g_user_lock);
}
/* what libxsmm_get_kernel_info / libxsmm_release_kernel need to know about a pointer that is not one of the thunks: is it the value
 * of a live user entry (returns 1 and its size), and release it (reference src/libxsmm_main.c: user entries ARE released) */
int xb_user_value_info(const void* value, size_t* size) {
  xb_user_entry* e; int found = 0;
  if (value == NULL) return 0;
  pthread_mutex_lock(&g_user_lock);
  e = user_of_value(value);
  if (e != NULL && e->dead == 0) { found = 1; if (size != NULL) *size = e->value_size; }
  pthread_mutex_unlock(&g_user_lock);
  return found;
}
int xb_user_value_release(const void* value) {
  xb_user_entry* e; int found = 0;
  if (value == NULL) return 0;
  pthread_mutex_lock(&g_user_lock);
  e = user_of_value(value);
  if (e != NULL && e->dead == 0) { e->dead = 1; found = 1; }
  pthread_mutex_unlock(&g_user_lock);
  return found;
}
/* enumeration of user entries: the first live entry, and the live entry after a given one (which may have been released meanwhile) */
void* xb_user_first(const void** key) {
  xb_user_entry* e; void* result = NULL;
  pthread_mutex_lock(&g_user_lock);
  for (e = g_user; e != NULL && e->dead != 0; e = e->next) {}
  if (e != NULL) { result = e->value; if (key != NULL) *key = e->key; }
  pthread_mutex_unlock(&g_user_lock);
  return result;
}
void* xb_user_next(const void* value, const void** key) {
  xb_user_entry* e; void* result = NULL;
  pthread_mutex_lock(&g_user_lock);
  e = user_of_value(value);
  if (e != NULL) for (e = e->next; e != NULL && e->dead != 0; e = e->next) {}
  if (e != NULL) { result = e->value; if (key != NULL) *key = e->key; }
  pthread_mutex_unlock(&g_user_lock);
  return result;
}
