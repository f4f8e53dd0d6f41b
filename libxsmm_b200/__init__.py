"""libxsmm_b200 -- Python mirror (ctypes) of the LIBXSMM-compatible C ABI exported by
``libxsmm_b200/lib/libxsmm_b200.so``.

The product is the C-ABI shared library (``include/*.h``); this module only binds it 1:1 so that the
parity tests and ``bench.py`` read like the reference's own drivers (same function names, argument
order and NULL-on-failure behaviour as ``include/libxsmm.h`` of the reference). PyTorch is used by the
callers for device memory and ``torch.distributed`` only -- nothing here computes anything, and
nothing here falls back to a CPU implementation: if the CUDA library is missing the import fails.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libxsmm_b200.so")
if not os.path.exists(LIB_PATH):
    raise ImportError(
        "libxsmm_b200: %s is missing -- build it with `make lib` (or __graft_entry__.build()); "
        "there is no CPU fallback" % LIB_PATH)
lib = C.CDLL(LIB_PATH)   # RTLD_LOCAL: the reference build used by the tests has same-named symbols

# ---- enumerations (include/libxsmm_typedefs.h) -------------------------------------------------------
_DT = ("F64 F32 BF16 F16 BF8 HF8 I64 U64 I32 U32 I16 U16 I8 U8 MXBF8 MXHF8 MXBF6 MXHF6 I4X2 U4X2 "
       "MXFP4X2 NVFP4X2 I2X4 I1X8 BF32 IMPLICIT UNSUPPORTED").split()
for _i, _n in enumerate(_DT):
    globals()["DATATYPE_" + _n] = _i
TYPESIZE = {0: 8, 1: 4, 2: 2, 3: 2, 4: 1, 5: 1, 6: 8, 7: 8, 8: 4, 9: 4, 10: 2, 11: 2, 12: 1, 13: 1, 14: 1, 15: 1, 18: 1, 19: 1, 20: 1, 22: 1, 23: 1, 24: 4}

GEMM_FLAG_NONE = 0
GEMM_FLAG_TRANS_A = 1
GEMM_FLAG_TRANS_B = 2
GEMM_FLAG_BETA_0 = 4
GEMM_FLAG_NO_RESET_TILECONFIG = 64
GEMM_FLAG_NO_SETUP_TILECONFIG = 128
GEMM_FLAG_VNNI_A = 256
GEMM_FLAG_VNNI_B = 512
GEMM_FLAG_VNNI_C = 1024
GEMM_PREFETCH_NONE = 0
GEMM_BATCH_REDUCE_NONE, GEMM_BATCH_REDUCE_ADDRESS, GEMM_BATCH_REDUCE_OFFSET, GEMM_BATCH_REDUCE_STRIDE = 0, 1, 2, 4

BACKEND_NONE, BACKEND_SIMT, BACKEND_TCGEN05, BACKEND_STREAM, BACKEND_NOOP = 0, 1, 2, 3, 4

_UNARY = ("NONE IDENTITY XOR X2 SQRT RELU RELU_INV TANH TANH_INV SIGMOID SIGMOID_INV GELU GELU_INV NEGATE INC "
          "RECIPROCAL RECIPROCAL_SQRT EXP REDUCE_X_OP_ADD REDUCE_X2_OP_ADD REDUCE_X_X2_OP_ADD REDUCE_X_OP_MAX "
          "REDUCE_X_OP_MUL REDUCE_X_OP_ADD_NCNC_FORMAT REDUCE_TO_SCALAR_OP_ADD DROPOUT DROPOUT_INV REPLICATE_COL_VAR "
          "TRANSFORM_NORM_TO_VNNI2 TRANSFORM_NORM_TO_NORMT TRANSFORM_VNNI2_TO_VNNI2T TRANSFORM_NORM_TO_VNNI2T "
          "TRANSFORM_NORM_TO_VNNI2_PAD UNZIP LEAKY_RELU LEAKY_RELU_INV ELU ELU_INV STOCHASTIC_ROUND TRANSFORM_PADM_MOD2 "
          "TRANSFORM_PADN_MOD2 TRANSFORM_PADNM_MOD2 QUANT DEQUANT REDUCE_COLS_IDX_OP_ADD DECOMPRESS_SPARSE_FACTOR_1 "
          "DECOMPRESS_SPARSE_FACTOR_2 DECOMPRESS_SPARSE_FACTOR_4 DECOMPRESS_SPARSE_FACTOR_8 DECOMPRESS_SPARSE_FACTOR_16 "
          "DECOMPRESS_SPARSE_FACTOR_32 GATHER SCATTER REDUCE_COLS_IDX_OP_MAX TRANSFORM_NORM_TO_VNNI4 "
          "TRANSFORM_VNNI4_TO_VNNI4T TRANSFORM_NORM_TO_VNNI4T TRANSFORM_NORM_TO_VNNI4_PAD TRANSFORM_PADM_MOD4 "
          "TRANSFORM_PADN_MOD4 TRANSFORM_PADNM_MOD4 TRANSFORM_VNNI4_TO_NORM TRANSFORM_VNNI4_TO_VNNI2 DUMP "
          "DECOMP_FP32_TO_BF16X2 DECOMP_FP32_TO_BF16X3 TRANSFORM_VNNI4T_TO_NORM TRANSFORM_VNNI2T_TO_NORM "
          "REDUCE_COLS_IDX_OP_MIN REDUCE_X_OP_MIN REDUCE_X_OP_ABSMAX TRANSFORM_NORM_TO_VNNI8 TRANSFORM_VNNI8_TO_VNNI8T "
          "TRANSFORM_NORM_TO_VNNI8T TRANSFORM_NORM_TO_VNNI8_PAD TRANSFORM_VNNI8T_TO_NORM TRANSFORM_VNNI8_TO_NORM").split()
for _i, _n in enumerate(_UNARY):
    globals()["MELTW_TYPE_UNARY_" + _n] = _i
_BINARY = ("NONE ADD MUL SUB DIV MULADD MATMUL MUL_AND_REDUCE_TO_SCALAR_OP_ADD PACK MAX MIN BRGEMM BRGEMM_B_TRANS "
           "BRGEMM_A_TRANS BRGEMM_A_TRANS_B_TRANS BRGEMM_A_VNNI BRGEMM_A_VNNI_B_TRANS BRGEMM_A_VNNI_TRANS "
           "BRGEMM_A_VNNI_TRANS_B_TRANS MATMUL_B_TRANS MATMUL_A_TRANS MATMUL_A_TRANS_B_TRANS MATMUL_A_VNNI "
           "MATMUL_A_VNNI_B_TRANS MATMUL_A_VNNI_TRANS MATMUL_A_VNNI_TRANS_B_TRANS ZIP CMP_OP_GT CMP_OP_GE CMP_OP_LT "
           "CMP_OP_LE CMP_OP_EQ CMP_OP_NE").split()
for _i, _n in enumerate(_BINARY):
    globals()["MELTW_TYPE_BINARY_" + _n] = _i
MELTW_TYPE_TERNARY_NONE, MELTW_TYPE_TERNARY_MULADD, MELTW_TYPE_TERNARY_MATMUL, MELTW_TYPE_TERNARY_SELECT, \
    MELTW_TYPE_TERNARY_NMULADD = 0, 1, 2, 3, 4

MELTW_FLAG_UNARY_NONE = 0
MELTW_FLAG_UNARY_BITMASK_2BYTEMULT = 1
MELTW_FLAG_UNARY_BCAST_ROW = 2
MELTW_FLAG_UNARY_BCAST_COL = 4
MELTW_FLAG_UNARY_BCAST_SCALAR = 8
MELTW_FLAG_UNARY_REDUCE_COLS = 16
MELTW_FLAG_UNARY_REDUCE_ROWS = 32
MELTW_FLAG_UNARY_REDUCE_INIT_ACC = 64
MELTW_FLAG_UNARY_IDX_SIZE_4BYTES = 128
MELTW_FLAG_UNARY_IDX_SIZE_8BYTES = 256
MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP = 2048
MELTW_FLAG_UNARY_GS_ROWS = 16
MELTW_FLAG_UNARY_GS_COLS = 32
MELTW_FLAG_UNARY_GS_OFFS = 8192
MELTW_FLAG_UNARY_NO_SCF_QUANT = 1024
MELTW_FLAG_UNARY_SIGN_SAT_QUANT = 16
MELTW_FLAG_UNARY_STOCHASTIC_ROUND = 4096
MELTW_FLAG_BINARY_NONE = 0
MELTW_FLAG_BINARY_BCAST_ROW_IN_0, MELTW_FLAG_BINARY_BCAST_ROW_IN_1 = 1, 2
MELTW_FLAG_BINARY_BCAST_COL_IN_0, MELTW_FLAG_BINARY_BCAST_COL_IN_1 = 4, 8
MELTW_FLAG_BINARY_BCAST_SCALAR_IN_0, MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1 = 16, 32
MELTW_FLAG_BINARY_BITMASK_2BYTEMULT = 128
MELTW_FLAG_BINARY_STOCHASTIC_ROUND = 64
MELTW_FLAG_TERNARY_NONE = 0
MELTW_FLAG_TERNARY_BCAST_ROW_IN_0, MELTW_FLAG_TERNARY_BCAST_ROW_IN_1, MELTW_FLAG_TERNARY_BCAST_ROW_IN_2 = 1, 2, 4
MELTW_FLAG_TERNARY_BCAST_COL_IN_0, MELTW_FLAG_TERNARY_BCAST_COL_IN_1, MELTW_FLAG_TERNARY_BCAST_COL_IN_2 = 8, 16, 32
MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_0, MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_1, MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_2 = 64, 128, 256
MELTW_FLAG_TERNARY_BITMASK_2BYTEMULT = 1024
MELTW_FLAG_TERNARY_STOCHASTIC_ROUND = 2048


# ---- structs (layouts of include/libxsmm_typedefs.h) --------------------------------------------------
class MatrixArg(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("primary", "secondary", "tertiary", "quaternary", "quinary", "senary")]


class MatrixOpArg(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("primary", "secondary", "tertiary", "quaternary")]


class GemmParam(C.Structure):
    _fields_ = [("op", MatrixOpArg), ("a", MatrixArg), ("b", MatrixArg), ("c", MatrixArg)]


class GemmExtParam(C.Structure):
    _fields_ = [("op", MatrixOpArg), ("a", MatrixArg), ("b", MatrixArg), ("c", MatrixArg), ("d", MatrixArg),
                ("ap", MatrixArg), ("bp", MatrixArg), ("cp", MatrixArg)]


class MeltwUnaryParam(C.Structure):
    _fields_ = [("op", MatrixOpArg), ("inp", MatrixArg), ("out", MatrixArg)]


class MeltwBinaryParam(C.Structure):
    _fields_ = [("op", MatrixOpArg), ("in0", MatrixArg), ("in1", MatrixArg), ("out", MatrixArg)]


class MeltwTernaryParam(C.Structure):
    _fields_ = [("op", MatrixOpArg), ("in0", MatrixArg), ("in1", MatrixArg), ("in2", MatrixArg), ("out", MatrixArg)]


class MeqnArgShape(C.Structure):
    _fields_ = [("m", C.c_int), ("n", C.c_int), ("ld", C.c_int), ("type", C.c_int)]


class MatrixArgAttributes(C.Structure):
    _fields_ = [("type", C.c_int), ("set_type", C.c_int), ("set_cardinality_hint", C.c_int), ("set_stride_hint", C.c_int)]


class MeqnMetadata(C.Structure):
    _fields_ = [("eqn_idx", C.c_int), ("pos", C.c_int)]


class MeqnParam(C.Structure):
    _fields_ = [("ops_args", C.c_void_p), ("inputs", C.c_void_p), ("output", MatrixArg)]


class GemmShape(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("m", "n", "k", "lda", "ldb", "ldc", "a_in_type", "b_in_type", "out_type", "comp_type")]


class BatchReduceConfig(C.Structure):
    _fields_ = [("br_type", C.c_int), ("br_stride_a_hint", C.c_int), ("br_stride_b_hint", C.c_int), ("br_unroll_hint", C.c_ubyte)]


class SpgemmConfig(C.Structure):
    _fields_ = [("packed_width", C.c_int), ("bk", C.c_int), ("bn", C.c_int)]


class GemmExtUnaryArgops(C.Structure):
    _fields_ = [("ldap", C.c_int), ("ap_unary_type", C.c_int), ("ap_unary_flags", C.c_uint), ("store_ap", C.c_int),
                ("ldbp", C.c_int), ("bp_unary_type", C.c_int), ("bp_unary_flags", C.c_uint), ("store_bp", C.c_int),
                ("ldcp", C.c_int), ("cp_unary_type", C.c_int), ("cp_unary_flags", C.c_uint), ("store_cp", C.c_int)]


class GemmExtBinaryPostops(C.Structure):
    _fields_ = [("ldd", C.c_int), ("d_in_type", C.c_int), ("d_binary_type", C.c_int), ("d_binary_flags", C.c_uint)]


class MeltwUnaryShape(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("m", "n", "ldi", "ldo", "in0_type", "out_type", "comp_type")]


class MeltwBinaryShape(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("m", "n", "ldi", "ldi2", "ldo", "in0_type", "in1_type", "out_type", "comp_type")]


class MeltwTernaryShape(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("m", "n", "ldi", "ldi2", "ldi3", "ldo", "in0_type", "in1_type", "in2_type",
                                      "out_type", "comp_type")]


class MMKernelInfo(C.Structure):
    _fields_ = [("iprecision", C.c_int), ("oprecision", C.c_int), ("prefetch", C.c_int), ("lda", C.c_uint), ("ldb", C.c_uint),
                ("ldc", C.c_uint), ("m", C.c_uint), ("n", C.c_uint), ("k", C.c_uint), ("flags", C.c_int)]


class KernelInfo(C.Structure):
    _fields_ = [("kind", C.c_int), ("nflops", C.c_uint), ("code_size", C.c_size_t), ("is_reference_kernel", C.c_uint)]


class RegistryInfo(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("capacity", "size", "nbytes", "nstatic", "ncache")]


GEMMFUNCTION = C.CFUNCTYPE(None, C.POINTER(GemmParam))
GEMMFUNCTION_EXT = C.CFUNCTYPE(None, C.POINTER(GemmExtParam))
TILECFGFUNCTION = C.CFUNCTYPE(None, C.c_void_p)
MELTW_UNARY_FN = C.CFUNCTYPE(None, C.POINTER(MeltwUnaryParam))
MELTW_BINARY_FN = C.CFUNCTYPE(None, C.POINTER(MeltwBinaryParam))
MELTW_TERNARY_FN = C.CFUNCTYPE(None, C.POINTER(MeltwTernaryParam))


def _sig(name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


# every symbol declared in include/libxsmm.h, include/libxsmm_fsspmdm.h and include/libxsmm_b200.h
_I, _U, _P, _LL, _ULL = C.c_int, C.c_uint, C.c_void_p, C.c_longlong, C.c_ulonglong
libxsmm_init = _sig("libxsmm_init", None, [])
libxsmm_finalize = _sig("libxsmm_finalize", None, [])
libxsmm_get_target_archid = _sig("libxsmm_get_target_archid", _I, [])
libxsmm_set_target_archid = _sig("libxsmm_set_target_archid", None, [_I])
libxsmm_get_target_arch = _sig("libxsmm_get_target_arch", C.c_char_p, [])
libxsmm_set_target_arch = _sig("libxsmm_set_target_arch", None, [C.c_char_p])
libxsmm_get_typename = _sig("libxsmm_get_typename", C.c_char_p, [_I])
libxsmm_typesize = _sig("libxsmm_typesize", C.c_ubyte, [_I])
libxsmm_get_verbosity = _sig("libxsmm_get_verbosity", _I, [])
libxsmm_set_verbosity = _sig("libxsmm_set_verbosity", None, [_I])
libxsmm_get_mmkernel_info = _sig("libxsmm_get_mmkernel_info", _I, [_P, C.POINTER(MMKernelInfo)])
libxsmm_get_kernel_info = _sig("libxsmm_get_kernel_info", _I, [_P, C.POINTER(KernelInfo)])
libxsmm_get_registry_info = _sig("libxsmm_get_registry_info", _I, [C.POINTER(RegistryInfo)])
libxsmm_get_registry_begin = _sig("libxsmm_get_registry_begin", _P, [_I, C.POINTER(_P)])
libxsmm_get_registry_next = _sig("libxsmm_get_registry_next", _P, [_P, C.POINTER(_P)])
libxsmm_create_gemm_shape = _sig("libxsmm_create_gemm_shape", GemmShape, [_I] * 10)
libxsmm_create_gemm_batch_reduce_config = _sig("libxsmm_create_gemm_batch_reduce_config", BatchReduceConfig, [_I, _I, _I, C.c_ubyte])
libxsmm_create_gemm_ext_unary_argops = _sig("libxsmm_create_gemm_ext_unary_argops", GemmExtUnaryArgops,
                                            [_I, _I, _U, _I, _I, _I, _U, _I, _I, _I, _U, _I])
libxsmm_create_gemm_ext_binary_postops = _sig("libxsmm_create_gemm_ext_binary_postops", GemmExtBinaryPostops, [_I, _I, _I, _U])
libxsmm_create_meltw_unary_shape = _sig("libxsmm_create_meltw_unary_shape", MeltwUnaryShape, [_I] * 7)
libxsmm_create_meltw_binary_shape = _sig("libxsmm_create_meltw_binary_shape", MeltwBinaryShape, [_I] * 9)
libxsmm_create_meltw_ternary_shape = _sig("libxsmm_create_meltw_ternary_shape", MeltwTernaryShape, [_I] * 11)
libxsmm_dispatch_gemm = _sig("libxsmm_dispatch_gemm", _P, [GemmShape, _U, _U])
libxsmm_dispatch_brgemm = _sig("libxsmm_dispatch_brgemm", _P, [GemmShape, _U, _U, BatchReduceConfig])
libxsmm_dispatch_brgemm_ext = _sig("libxsmm_dispatch_brgemm_ext", _P,
                                   [GemmShape, _U, _U, BatchReduceConfig, GemmExtUnaryArgops, GemmExtBinaryPostops])
libxsmm_dispatch_tilecfg_gemm = _sig("libxsmm_dispatch_tilecfg_gemm", _P, [GemmShape, _U])
libxsmm_dispatch_meltw_unary = _sig("libxsmm_dispatch_meltw_unary", _P, [_I, MeltwUnaryShape, _U])
libxsmm_dispatch_meltw_binary = _sig("libxsmm_dispatch_meltw_binary", _P, [_I, MeltwBinaryShape, _U])
libxsmm_dispatch_meltw_ternary = _sig("libxsmm_dispatch_meltw_ternary", _P, [_I, MeltwTernaryShape, _U])
libxsmm_meqn_create = _sig("libxsmm_meqn_create", _I, [])
libxsmm_create_meqn_arg_shape = _sig("libxsmm_create_meqn_arg_shape", MeqnArgShape, [_I, _I, _I, _I])
libxsmm_create_matrix_arg_attributes = _sig("libxsmm_create_matrix_arg_attributes", MatrixArgAttributes, [_I, _I, _I, _I])
libxsmm_create_meqn_arg_metadata = _sig("libxsmm_create_meqn_arg_metadata", MeqnMetadata, [_I, _I])
libxsmm_create_meqn_op_metadata = _sig("libxsmm_create_meqn_op_metadata", MeqnMetadata, [_I, _I])
libxsmm_meqn_push_back_arg = _sig("libxsmm_meqn_push_back_arg", _I, [MeqnMetadata, MeqnArgShape, MatrixArgAttributes])
libxsmm_meqn_push_back_unary_op = _sig("libxsmm_meqn_push_back_unary_op", _I, [MeqnMetadata, _I, _I, _U])
libxsmm_meqn_push_back_binary_op = _sig("libxsmm_meqn_push_back_binary_op", _I, [MeqnMetadata, _I, _I, _U])
libxsmm_meqn_push_back_ternary_op = _sig("libxsmm_meqn_push_back_ternary_op", _I, [MeqnMetadata, _I, _I, _U])
libxsmm_dispatch_meqn = _sig("libxsmm_dispatch_meqn", _P, [_I, MeqnArgShape])
MEQN_FN = C.CFUNCTYPE(None, C.POINTER(MeqnParam))
libxsmm_xregister = _sig("libxsmm_xregister", _P, [_P, C.c_size_t, C.c_size_t, _P])
libxsmm_xdispatch = _sig("libxsmm_xdispatch", _P, [_P, C.c_size_t])
libxsmm_xrelease = _sig("libxsmm_xrelease", None, [_P, C.c_size_t])
libxsmm_create_packed_gemm = _sig("libxsmm_create_packed_gemm", _P, [GemmShape, _U, _U, _I])
libxsmm_create_packed_gemm_ac_rm = _sig("libxsmm_create_packed_gemm_ac_rm", _P, [GemmShape, _U, _U, _I])
libxsmm_create_packed_gemm_bc_rm = _sig("libxsmm_create_packed_gemm_bc_rm", _P, [GemmShape, _U, _U, _I])
libxsmm_create_packed_spgemm_csr = _sig("libxsmm_create_packed_spgemm_csr", _P, [GemmShape, _U, _U, _I, _P, _P, _P])
libxsmm_create_packed_spgemm_csc = _sig("libxsmm_create_packed_spgemm_csc", _P, [GemmShape, _U, _U, _I, _P, _P, _P])
libxsmm_create_packed_spgemm_bcsc = _sig("libxsmm_create_packed_spgemm_bcsc", _P, [GemmShape, _U, _U, SpgemmConfig])
libxsmm_create_tilecfg_packed_spgemm_bcsc = _sig("libxsmm_create_tilecfg_packed_spgemm_bcsc", _P, [GemmShape, _U, SpgemmConfig])
libxsmm_create_spgemm_csr_areg = _sig("libxsmm_create_spgemm_csr_areg", _P, [GemmShape, _U, _U, _I, _P, _P, _P])
libxsmm_release_kernel = _sig("libxsmm_release_kernel", None, [_P])
# BLAS-style GEMM: every argument by reference (char*, blasint*, scalar*), a/b/c as addresses
libxsmm_dgemm = _sig("libxsmm_dgemm", None, [C.c_char_p, C.c_char_p, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P])
libxsmm_sgemm = _sig("libxsmm_sgemm", None, [C.c_char_p, C.c_char_p, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P])
libxsmm_malloc = _sig("libxsmm_malloc", _P, [C.c_size_t])
libxsmm_aligned_malloc = _sig("libxsmm_aligned_malloc", _P, [C.c_size_t, C.c_size_t])
libxsmm_free = _sig("libxsmm_free", None, [_P])
libxsmm_convert_bf16_to_f32 = _sig("libxsmm_convert_bf16_to_f32", C.c_float, [C.c_ushort])
libxsmm_convert_f16_to_f32 = _sig("libxsmm_convert_f16_to_f32", C.c_float, [C.c_ushort])
libxsmm_convert_f32_to_bf16_rne = _sig("libxsmm_convert_f32_to_bf16_rne", C.c_ushort, [C.c_float])
libxsmm_convert_f32_to_f16 = _sig("libxsmm_convert_f32_to_f16", C.c_ushort, [C.c_float])
libxsmm_fsspmdm_create = _sig("libxsmm_fsspmdm_create", _P, [_I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _I, _P])
libxsmm_dfsspmdm_create = _sig("libxsmm_dfsspmdm_create", _P, [_I, _I, _I, _I, _I, _I, C.c_double, C.c_double, _P, _I, _P])
libxsmm_sfsspmdm_create = _sig("libxsmm_sfsspmdm_create", _P, [_I, _I, _I, _I, _I, _I, C.c_float, C.c_float, _P, _I, _P])
libxsmm_fsspmdm_execute = _sig("libxsmm_fsspmdm_execute", None, [_P, _P, _P])
libxsmm_dfsspmdm_execute = _sig("libxsmm_dfsspmdm_execute", None, [_P, _P, _P])
libxsmm_sfsspmdm_execute = _sig("libxsmm_sfsspmdm_execute", None, [_P, _P, _P])
libxsmm_fsspmdm_destroy = _sig("libxsmm_fsspmdm_destroy", None, [_P])
libxsmm_dfsspmdm_destroy = _sig("libxsmm_dfsspmdm_destroy", None, [_P])
libxsmm_sfsspmdm_destroy = _sig("libxsmm_sfsspmdm_destroy", None, [_P])
# additive GPU entry points (include/libxsmm_b200.h)
libxsmm_b200_device_count = _sig("libxsmm_b200_device_count", _I, [])
libxsmm_b200_set_device = _sig("libxsmm_b200_set_device", _I, [_I])
libxsmm_b200_set_stream = _sig("libxsmm_b200_set_stream", None, [_P])
libxsmm_b200_set_blocking = _sig("libxsmm_b200_set_blocking", None, [_I])
libxsmm_b200_sync = _sig("libxsmm_b200_sync", _I, [])
libxsmm_b200_last_error = _sig("libxsmm_b200_last_error", _I, [])
libxsmm_b200_last_error_string = _sig("libxsmm_b200_last_error_string", C.c_char_p, [])
libxsmm_b200_launch_count = _sig("libxsmm_b200_launch_count", _ULL, [])
libxsmm_b200_launch_count_backend = _sig("libxsmm_b200_launch_count_backend", _ULL, [_I])
libxsmm_b200_kernel_backend = _sig("libxsmm_b200_kernel_backend", _I, [_P])
libxsmm_b200_bcsc_variant = _sig("libxsmm_b200_bcsc_variant", _I, [_P, _ULL])
libxsmm_b200_fsspmdm_variant = _sig("libxsmm_b200_fsspmdm_variant", _I, [_P, _P, _P])
libxsmm_b200_meltw_variant = _sig("libxsmm_b200_meltw_variant", _I, [_P, _P])
libxsmm_b200_set_force_simt = _sig("libxsmm_b200_set_force_simt", None, [_I])
libxsmm_b200_device_malloc = _sig("libxsmm_b200_device_malloc", _P, [C.c_size_t])
libxsmm_b200_device_free = _sig("libxsmm_b200_device_free", None, [_P])
libxsmm_b200_host_malloc = _sig("libxsmm_b200_host_malloc", _P, [C.c_size_t])
libxsmm_b200_host_free = _sig("libxsmm_b200_host_free", None, [_P])
libxsmm_b200_memcpy = _sig("libxsmm_b200_memcpy", _I, [_P, _P, C.c_size_t])
libxsmm_b200_gemm_batch_strided = _sig("libxsmm_b200_gemm_batch_strided", _I, [_P, _P, _P, _P, _LL, _LL, _LL, _ULL, _LL])
libxsmm_b200_gemm_batch_strided_scaled = _sig("libxsmm_b200_gemm_batch_strided_scaled", _I,
                                              [_P, _P, _P, _P, _LL, _LL, _LL, _P, _P, _P, _LL, _LL, _LL, _ULL, _LL])
libxsmm_b200_gemm_batch_strided_multi = _sig("libxsmm_b200_gemm_batch_strided_multi", _I, [_P, _P, _P, _P, _LL, _LL, _LL, _ULL, _LL, _I])
libxsmm_b200_gemm_batch_grid = _sig("libxsmm_b200_gemm_batch_grid", _I, [_P, _P, _P, _P, _LL, _LL, _LL, _LL, _ULL, _LL, _LL])
libxsmm_b200_gemm_batch = _sig("libxsmm_b200_gemm_batch", _I, [_P, C.POINTER(GemmParam), _LL])
libxsmm_b200_gemm_plan_create = _sig("libxsmm_b200_gemm_plan_create", _P, [_P, C.POINTER(GemmParam), _LL])
libxsmm_b200_gemm_plan_run = _sig("libxsmm_b200_gemm_plan_run", _I, [_P])
libxsmm_b200_gemm_plan_destroy = _sig("libxsmm_b200_gemm_plan_destroy", None, [_P])
libxsmm_b200_gemm_plan_is_pooled = _sig("libxsmm_b200_gemm_plan_is_pooled", _I, [_P])


class MeltwStrides(C.Structure):
    _fields_ = [(n, C.c_longlong) for n in ("in0", "in1", "in2", "in_aux", "out", "out_aux")]


libxsmm_b200_meltw_batch_strided = _sig("libxsmm_b200_meltw_batch_strided", _I, [_P, _P, C.POINTER(MeltwStrides), _LL])
libxsmm_b200_meqn_batch_strided = _sig("libxsmm_b200_meqn_batch_strided", _I,
                                       [_P, C.POINTER(MeqnParam), C.POINTER(_LL), _LL, _LL, C.POINTER(_LL), _LL])


class SpgemmStrides(C.Structure):
    _fields_ = [(n, C.c_longlong) for n in ("a", "b", "c")]


libxsmm_b200_spgemm_batch_strided = _sig("libxsmm_b200_spgemm_batch_strided", _I, [_P, C.POINTER(GemmParam), C.POINTER(SpgemmStrides), _LL])


class GemmExtStrides(C.Structure):
    _fields_ = [(n, C.c_longlong) for n in ("a", "b", "c", "bias", "mask")]


libxsmm_b200_gemm_ext_batch_strided = _sig("libxsmm_b200_gemm_ext_batch_strided", _I, [_P, C.POINTER(GemmExtParam), C.POINTER(GemmExtStrides), _LL])
libxsmm_b200_gemm_ext_batch = _sig("libxsmm_b200_gemm_ext_batch", _I, [_P, C.POINTER(GemmExtParam), _LL])

EXPORTED = [n for n in dir() if n.startswith("libxsmm_") and callable(globals()[n])]


# ---- small conveniences used by tests and bench.py -----------------------------------------------------
def ptr(x):
    """Raw address of a torch tensor, numpy array, ctypes object or int."""
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if hasattr(x, "ctypes"):
        return x.ctypes.data
    if isinstance(x, int):
        return x
    return C.addressof(x)


def call_gemm(kernel, a, b, c, br_count=None, a_aux=None, b_aux=None, scf=None, colptr=None, rowidx=None, nblocks=None,
              a_scales=None, b_scales=None, c_scales=None, a_zero_points=None):
    """Invoke a GEMM-family handle like the reference drivers do (fill libxsmm_gemm_param, call).
    a_scales / b_scales / c_scales: the E8M0 block scales of an MX handle (a/b/c.tertiary); a_scales is also the m row scales of a
    dequantising A (I8 x BF16: f32, I8 / I4 / U4 x F16: f16), and a_zero_points the m f16 zero points of an int4 A (a.quaternary);
    for MXFP4 x I8, a_scales / b_scales are A's E8M0 and B's f32 block scales."""
    p = GemmParam()
    keep = []
    if br_count is not None:
        brc = C.c_ulonglong(br_count)
        keep.append(brc)
        p.op.tertiary = C.addressof(brc)
    p.a.primary, p.b.primary, p.c.primary = ptr(a), ptr(b), ptr(c)
    if a_aux is not None:
        p.a.secondary = ptr(a_aux)
    if b_aux is not None:
        p.b.secondary = ptr(b_aux)
    if scf is not None:
        s = C.c_float(scf)
        keep.append(s)
        p.c.tertiary = C.addressof(s)
    if colptr is not None:
        p.b.secondary = ptr(colptr)
        p.b.tertiary = ptr(rowidx)
        nb = C.c_ulonglong(nblocks)
        keep.append(nb)
        p.b.quaternary = C.addressof(nb)
    if a_scales is not None:
        p.a.tertiary = ptr(a_scales)
    if b_scales is not None:
        p.b.tertiary = ptr(b_scales)
    if c_scales is not None:
        p.c.tertiary = ptr(c_scales)
    if a_zero_points is not None:
        p.a.quaternary = ptr(a_zero_points)
    GEMMFUNCTION(kernel)(C.byref(p))
    return keep


def check():
    """Raise if a kernel launched by this library failed (handles themselves return void)."""
    rc = libxsmm_b200_sync()
    if rc != 0:
        raise RuntimeError("libxsmm_b200: CUDA error %d: %s" % (rc, libxsmm_b200_last_error_string().decode()))
