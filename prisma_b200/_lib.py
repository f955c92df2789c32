"""ctypes binding of libprisma_b200.so (the C ABI in include/prisma_b200.h).

There is deliberately no fallback: if the CUDA library is missing or fails to load, importing a
band engine raises.  Only this module touches ctypes; everything else goes through `lib()`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PRISMA_B200_LIB") or os.path.join(_HERE, "libprisma_b200.so")  # override: an instrumented build
_lib = None

c_float_p = C.POINTER(C.c_float)
c_u8_p = C.POINTER(C.c_uint8)
c_i64_p = C.POINTER(C.c_int64)
c_double_p = C.POINTER(C.c_double)


class DebugEpilogue(C.Structure):
    """Mirror of `prisma_debug_epilogue` (include/prisma_b200.h): pointer fields take device addresses (ints)."""
    _fields_ = [
        ("size", C.c_int), ("alpha", C.c_float), ("bias", C.c_void_p), ("gamma", C.c_void_p), ("act", C.c_int),
        ("pre_f32", C.c_void_p), ("pre_f32_ld", C.c_int), ("res_f32", C.c_void_p), ("res_f32_ld", C.c_int),
        ("res_a", C.c_void_p), ("res_a_ld", C.c_int), ("res_b", C.c_void_p), ("res_b_ld", C.c_int),
        ("out_f32", C.c_void_p), ("out_f32_ld", C.c_int), ("out_f16", C.c_void_p), ("out_f16_ld", C.c_int),
        ("out_f16_relu", C.c_void_p), ("out_f16_relu_ld", C.c_int),
        ("row_map", C.c_int), ("img_rows", C.c_int), ("in_w", C.c_int), ("in_h", C.c_int), ("out_wp", C.c_int),
        ("out_img_rows", C.c_int), ("sub", C.c_int), ("pad", C.c_int), ("out_pad", C.c_int), ("lead", C.c_int),
        ("out_lead", C.c_int), ("shuf_s", C.c_int), ("shuf_cout", C.c_int),
        ("head_w", C.c_void_p), ("head_b", C.c_float), ("head_out", C.c_void_p), ("stat_part", C.c_void_p),
        ("m_dev", C.c_void_p), ("tma_store", C.c_int),
        ("gru", C.c_int), ("gru_h", C.c_void_p), ("gru_z", C.c_void_p), ("gru_rh", C.c_void_p), ("gru_rh_ld", C.c_int),
    ]

    def __init__(self, **kw):
        defaults = dict(size=C.sizeof(DebugEpilogue), alpha=1.0, sub=1, pad=1, out_pad=1, lead=-1, out_lead=-1, shuf_s=1)
        defaults.update(kw)
        super().__init__(**defaults)

# name -> (restype, argtypes); must list every symbol declared in include/prisma_b200.h
SIGNATURES = {
    "prisma_last_error": (C.c_char_p, []),
    "prisma_device_count": (C.c_int, []),
    "prisma_version": (C.c_char_p, []),
    "prisma_depth_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "prisma_depth_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, c_i64_p, C.c_int]),
    "prisma_depth_finalize": (C.c_int, [C.c_void_p]),
    "prisma_depth_infer": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, c_float_p, c_u8_p, c_float_p, c_float_p]),
    "prisma_depth_infer_batch": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, C.c_int, c_float_p, c_u8_p, c_float_p, c_float_p]),
    "prisma_depth_infer_stream": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p, c_u8_p, c_float_p, c_float_p]),
    "prisma_host_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "prisma_host_free": (C.c_int, [C.c_void_p]),
    "prisma_depth_infer_resident": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_depth_encode": (C.c_int, [C.c_void_p, c_float_p, C.c_int, C.c_int, C.c_int, c_u8_p, c_float_p, c_float_p]),
    "prisma_depth_encode_png": (C.c_int, [C.c_void_p, c_float_p, C.c_int, C.c_int, C.c_int, c_u8_p, c_float_p, c_float_p]),
    "prisma_depth_infer_image": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, c_float_p, c_u8_p, c_float_p, c_float_p]),
    "prisma_depth_point_cloud": (C.c_int, [C.c_void_p, c_float_p, C.c_int, C.c_int, C.c_int, c_u8_p, c_u8_p]),
    "prisma_depth_set_net_side": (C.c_int, [C.c_void_p, C.c_int]),
    "prisma_depth_read_tap": (C.c_longlong, [C.c_void_p, C.c_char_p, c_float_p, C.c_longlong]),
    "prisma_depth_profile": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_depth_work": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, c_double_p]),
    "prisma_engine_destroy": (C.c_int, [C.c_void_p]),
    "prisma_flow_preprocess": (C.c_int, [C.c_int, c_u8_p, C.c_int, C.c_int, C.c_double, c_u8_p, c_float_p]),
    "prisma_flow_encode": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, c_u8_p, c_float_p]),
    "prisma_mask_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "prisma_mask_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, c_i64_p, C.c_int]),
    "prisma_mask_finalize": (C.c_int, [C.c_void_p]),
    "prisma_mask_infer": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, C.c_float, c_u8_p, C.POINTER(C.c_int), c_float_p,
                                    C.POINTER(C.c_int32), c_u8_p, c_float_p]),
    "prisma_mask_inject_feat": (C.c_int, [C.c_void_p, C.c_int, c_float_p, C.c_int, C.c_int]),
    "prisma_mask_infer_from_feats": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_u8_p, C.POINTER(C.c_int), c_float_p,
                                               C.POINTER(C.c_int32), c_u8_p]),
    "prisma_net_size": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "prisma_mask_sdf": (C.c_int, [C.c_int, c_u8_p, C.c_int, C.c_int, c_u8_p]),
    "prisma_mask_read_tap": (C.c_longlong, [C.c_void_p, C.c_char_p, c_float_p, C.c_longlong]),
    "prisma_mask_work": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_double)]),
    "prisma_flow_masks": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, c_u8_p, c_u8_p, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)]),
    "prisma_flowcorr_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "prisma_flowcorr_set_fmaps": (C.c_int, [C.c_void_p, c_float_p, c_float_p]),
    "prisma_flowcorr_build": (C.c_int, [C.c_void_p, C.c_int, c_float_p]),
    "prisma_flowcorr_lookup": (C.c_int, [C.c_void_p, c_float_p, c_float_p, C.c_int, c_float_p]),
    "prisma_flowcorr_read_level": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_flowcorr_work": (C.c_int, [C.c_void_p, c_double_p]),
    "prisma_flowcorr_create_pairs": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "prisma_flowcorr_set_frames": (C.c_int, [C.c_void_p, c_float_p]),
    "prisma_flow_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "prisma_flow_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, c_i64_p, C.c_int]),
    "prisma_flow_finalize": (C.c_int, [C.c_void_p]),
    "prisma_flow_infer": (C.c_int, [C.c_void_p, c_u8_p, c_u8_p, C.c_int, C.c_int, C.c_double, C.c_int, c_float_p, c_float_p,
                                    c_u8_p, c_u8_p, c_float_p, c_float_p, c_float_p]),
    "prisma_flow_infer_video": (C.c_int, [C.c_void_p, c_u8_p, c_u8_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, c_float_p,
                                          c_float_p, c_u8_p, c_u8_p, c_float_p, c_float_p, c_float_p]),
    "prisma_flow_read_tap": (C.c_longlong, [C.c_void_p, C.c_char_p, c_float_p, C.c_longlong]),
    "prisma_flow_work": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, c_double_p]),
    "prisma_flow_work_detail": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, c_double_p]),
    "prisma_flow_profile": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, c_float_p]),
    "prisma_flow_infer_stream": (C.c_int, [C.c_void_p, c_u8_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, c_float_p,
                                           c_float_p, c_u8_p, c_u8_p, c_float_p, c_float_p, C.POINTER(C.c_int)]),
    "prisma_flow_set_pairs_per_pass": (C.c_int, [C.c_void_p, C.c_int]),
    "prisma_flow_pairs_per_pass": (C.c_int, [C.c_void_p]),
    "prisma_flow_plan_pairs": (C.c_int, [C.c_void_p]),
    "prisma_flow_infer_resident": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_gemm": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_gemm_tf32x3": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, c_float_p]),
    "prisma_debug_gemm_ep": (C.c_int, [C.c_int, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.POINTER(DebugEpilogue)]),
    "prisma_debug_conv": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_attention": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_attention_batch": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_layernorm": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int]),
    "prisma_debug_layernorm_skip": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int]),
    "prisma_debug_pos_embed": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_patchify": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_readout_concat": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_upsample_ac": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                           c_float_p, c_float_p]),
    "prisma_debug_upsample_bicubic": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, c_float_p, C.c_int, C.c_int]),
    "prisma_debug_da_preprocess": (C.c_int, [C.c_int, c_u8_p, C.c_int, C.c_int, c_float_p, C.c_int, C.c_int]),
    "prisma_debug_raft_stem_im2col": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_instnorm_stats": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_instnorm_slab_stats": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_instnorm_apply": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                              c_float_p, c_float_p, c_float_p]),
    "prisma_debug_raft_gru_operands": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int),
                                                 c_float_p, c_float_p, c_float_p, c_float_p, c_float_p]),
    "prisma_debug_raft_flow_im2col": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "prisma_debug_raft_flow_head2": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, c_float_p,
                                               c_float_p]),
    "prisma_debug_raft_convex_upsample": (C.c_int, [C.c_int, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                                                    C.c_int, C.c_int, C.c_int, C.c_int, c_float_p]),
}


class PrismaError(RuntimeError):
    pass


def lib():
    """Load (once) and return the shared library; raises if it is not built -- no CPU fallback exists."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PrismaError(f"{LIB_PATH} is not built: run `python -m prisma_b200.build` (needs nvcc). "
                              "prisma_b200 has no non-CUDA path.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc):
    if rc < 0:
        raise PrismaError(lib().prisma_last_error().decode() or f"prisma_b200 error {rc}")
    return rc


def fptr(a):
    """float32 C-contiguous numpy array -> float* (None passes NULL)."""
    if a is None:
        return None
    if a.dtype.name != "float32" or not a.flags["C_CONTIGUOUS"]:
        raise PrismaError(f"expected a C-contiguous float32 array, got {a.dtype} (contiguous={a.flags['C_CONTIGUOUS']})")
    return a.ctypes.data_as(c_float_p)


def u8ptr(a):
    if a is None:
        return None
    if a.dtype.name != "uint8" or not a.flags["C_CONTIGUOUS"]:
        raise PrismaError(f"expected a C-contiguous uint8 array, got {a.dtype}")
    return a.ctypes.data_as(c_u8_p)
