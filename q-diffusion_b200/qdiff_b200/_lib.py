"""ctypes binding of libqdiff_b200.so (C ABI declared in include/qdiff_b200.h).

The structures below mirror the header field by field.  There is NO CPU fallback: if the
shared library is missing the import of any compute entry point raises, and every call that
needs a GPU fails loudly with the library's own error text.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# QDIFF_B200_LIB: another build of the same library (A/B timing of kernel variants); the default is the in-tree build
LIB_PATH = os.environ.get("QDIFF_B200_LIB") or os.path.join(_HERE, "libqdiff_b200.so")

c_ll = C.c_longlong
c_i32 = C.c_int32
c_f = C.c_float
c_vp = C.c_void_p

QD_OP_GEMM, QD_OP_QUANTIZE, QD_OP_GROUPNORM, QD_OP_LAYERNORM, QD_OP_IM2COL, QD_OP_ATTENTION = 1, 2, 3, 4, 5, 6
QD_OP_TIMESTEP_EMB, QD_OP_COPY2D, QD_OP_NCHW_TO_NHWC, QD_OP_NHWC_TO_NCHW, QD_OP_AVGPOOL2X, QD_OP_UPSAMPLE2X = 7, 8, 9, 10, 11, 12
QD_OP_SPLIT3, QD_OP_ATTENTION_FP, QD_OP_VQ_LOOKUP, QD_OP_SOFTMAX_ROWS, QD_OP_EMBED = 13, 14, 15, 16, 17


class QParams(C.Structure):
    _fields_ = [("delta", c_f), ("zero_point", c_i32), ("qmin", c_i32), ("qmax", c_i32)]


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", c_vp), ("w", c_vp), ("lda", c_ll),
        ("M", c_i32), ("N", c_i32), ("C", c_i32), ("taps", c_i32),
        ("w_rows", c_i32), ("B", c_i32), ("H", c_i32), ("W", c_i32),
        ("a_signed", c_i32),
        ("scale", c_vp), ("bias", c_vp), ("corr", c_vp), ("rowvec", c_vp),
        ("ld_rowvec", c_ll), ("rows_per_batch", c_i32), ("out_q_transposed", c_i32),
        ("residual", c_vp), ("ldr", c_ll),
        ("out", c_vp), ("ldo", c_ll),
        ("out_q", c_vp), ("ldq", c_ll),
        ("oq", QParams),
        ("bn_hint", c_i32), ("out_q_head_dim", c_i32), ("out_q_head_pitch", c_i32), ("geglu", c_i32),
        ("w_int4_packed", c_i32), ("k_dup", c_i32), ("w_zero", c_vp),
        ("scale_q", c_vp), ("bias_q", c_vp),
        ("gn_stats", c_vp), ("ld_stats", c_ll),
        ("a_bf16", c_i32), ("out_q_f16", c_i32),
    ]


class QuantizeDesc(C.Structure):
    _fields_ = [
        ("src", c_vp), ("ld_src", c_ll), ("dst", c_vp), ("ld_dst", c_ll),
        ("M", c_i32), ("C", c_i32), ("act", c_i32), ("split", c_i32),
        ("q0", QParams), ("q1", QParams),
        ("upsample2x", c_i32), ("B", c_i32), ("H", c_i32), ("W", c_i32),
    ]


class GroupNormDesc(C.Structure):
    _fields_ = [
        ("x", c_vp), ("ld_x", c_ll),
        ("B", c_i32), ("HW", c_i32), ("C", c_i32), ("groups", c_i32),
        ("eps", c_f), ("silu", c_i32),
        ("gamma", c_vp), ("beta", c_vp), ("ss_scale", c_vp), ("ss_shift", c_vp), ("ld_ss", c_ll),
        ("n_out", c_i32), ("reserved", c_i32),
        ("out_q", c_vp * 3), ("ld_q", c_ll * 3), ("q", QParams * 3),
        ("out_f", c_vp), ("ld_f", c_ll), ("ws", c_vp),
        ("raw_q", c_vp), ("ld_raw", c_ll), ("raw_split", c_i32), ("reserved2", c_i32), ("q_raw", QParams * 2),
        ("stats_in", c_vp), ("ld_stats_in", c_ll),
    ]


class LayerNormDesc(C.Structure):
    _fields_ = [
        ("x", c_vp), ("ld_x", c_ll), ("M", c_i32), ("C", c_i32), ("eps", c_f), ("n_out", c_i32),
        ("gamma", c_vp), ("beta", c_vp),
        ("out_q", c_vp * 3), ("ld_q", c_ll * 3), ("q", QParams * 3),
        ("out_f", c_vp), ("ld_f", c_ll),
    ]


class Im2colDesc(C.Structure):
    _fields_ = [
        ("src", c_vp), ("dst", c_vp), ("ld_dst", c_ll),
        ("B", c_i32), ("H", c_i32), ("W", c_i32), ("C", c_i32),
        ("Ho", c_i32), ("Wo", c_i32), ("stride", c_i32), ("pad_top", c_i32), ("pad_left", c_i32),
        ("pad_code", c_i32),
    ]


class AttentionDesc(C.Structure):
    _fields_ = [
        ("q", c_vp), ("k", c_vp), ("vt", c_vp),
        ("ld_q", c_ll), ("ld_k", c_ll), ("ld_vt", c_ll), ("v_batch_stride", c_ll),
        ("B", c_i32), ("heads", c_i32), ("d", c_i32), ("Tq", c_i32), ("Tk", c_i32),
        ("q_off", c_i32), ("k_off", c_i32), ("v_off", c_i32),
        ("head_stride_q", c_i32), ("head_stride_k", c_i32), ("head_stride_v", c_i32),
        ("q_signed", c_i32), ("k_signed", c_i32), ("v_signed", c_i32), ("p_signed", c_i32),
        ("zq", c_i32), ("zk", c_i32), ("zv", c_i32), ("zw", c_i32),
        ("p_qmin", c_i32), ("p_qmax", c_i32), ("sm_bits", c_i32),
        ("sim_scale", c_f), ("delta_w", c_f), ("out_scale", c_f),
        ("out", c_vp), ("ld_out", c_ll), ("ws", c_vp),
        ("out_q", c_vp), ("ld_out_q", c_ll), ("oq", QParams),
        ("qk_f16", c_i32), ("reserved5", c_i32),
    ]


class SplitDesc(C.Structure):
    _fields_ = [("src", c_vp), ("ld_src", c_ll), ("dst", c_vp), ("ld_dst", c_ll),
                ("M", c_i32), ("C", c_i32), ("Cp", c_i32), ("act", c_i32),
                ("upsample2x", c_i32), ("B", c_i32), ("H", c_i32), ("W", c_i32)]


class AttentionFpDesc(C.Structure):
    _fields_ = [("q", c_vp), ("k", c_vp), ("v", c_vp), ("ld_q", c_ll), ("ld_k", c_ll), ("ld_v", c_ll),
                ("B", c_i32), ("heads", c_i32), ("d", c_i32), ("Tq", c_i32), ("Tk", c_i32),
                ("q_off", c_i32), ("k_off", c_i32), ("v_off", c_i32),
                ("head_stride_q", c_i32), ("head_stride_k", c_i32), ("head_stride_v", c_i32),
                ("scale", c_f), ("out", c_vp), ("ld_out", c_ll), ("causal", c_i32)]


class EmbedDesc(C.Structure):
    _fields_ = [("ids", c_vp), ("tok", c_vp), ("pos", c_vp), ("out", c_vp), ("ld_out", c_ll),
                ("B", c_i32), ("T", c_i32), ("C", c_i32), ("vocab", c_i32)]


class MiscDesc(C.Structure):
    _fields_ = [("src", c_vp), ("dst", c_vp), ("ld_src", c_ll), ("ld_dst", c_ll),
                ("a", c_i32), ("b", c_i32), ("c", c_i32), ("d", c_i32), ("aux", c_vp)]


class SamplerDesc(C.Structure):
    _fields_ = [
        ("x", c_vp), ("eps", c_vp), ("old1", c_vp), ("old2", c_vp), ("old3", c_vp), ("noise", c_vp),
        ("x_prev", c_vp), ("pred_x0", c_vp), ("eps_out", c_vp),
        ("n", c_ll), ("cfg_scale", c_f),
        ("c_e0", c_f), ("c_e1", c_f), ("c_e2", c_f), ("c_e3", c_f),
        ("sqrt_at", c_f), ("sqrt_one_minus_at", c_f), ("sqrt_a_prev", c_f), ("dir_coef", c_f), ("sigma", c_f),
    ]


class AncestralDesc(C.Structure):
    _fields_ = [
        ("x", c_vp), ("eps", c_vp), ("noise", c_vp), ("x_prev", c_vp), ("pred_x0", c_vp),
        ("n", c_ll), ("c_x", c_f), ("c_e", c_f), ("m_x0", c_f), ("m_x", c_f), ("sigma", c_f), ("clamp", c_i32),
    ]


class WsearchDesc(C.Structure):
    _fields_ = [("w", c_vp), ("ld", c_ll), ("N", c_i32), ("k0", c_i32), ("k1", c_i32), ("n_bits", c_i32),
                ("delta", c_vp), ("zero_point", c_vp), ("index", c_vp), ("score", c_vp)]


EXPORTS = [
    "qd_qgemm_i8", "qd_quantize", "qd_groupnorm_quant", "qd_groupnorm_workspace_floats", "qd_layernorm_quant",
    "qd_im2col_i8", "qd_qattention", "qd_split_bf16x3", "qd_attention_fp32", "qd_embed_tokens", "qd_lincomb3", "qd_timestep_embedding", "qd_copy2d", "qd_nchw_to_nhwc", "qd_nhwc_to_nchw", "qd_avgpool2x", "qd_upsample2x_f32", "qd_vq_lookup", "qd_softmax_rows",
    "qd_sampler_step", "qd_ancestral_step", "qd_weight_scale_search", "qd_engine_create", "qd_engine_add_op", "qd_engine_num_ops", "qd_engine_finalize",
    "qd_engine_run", "qd_engine_run_range", "qd_engine_destroy", "qd_last_error", "qd_num_sms", "qd_launch_count",
]

_lib = None


def lib():
    """Load the shared library (once).  Raises if it has not been built: no fallback path exists."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"qdiff_b200: {LIB_PATH} is missing. Build it with `python __graft_entry__.py` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        getattr(L, name)  # raises AttributeError when a declared symbol is not exported
    L.qd_last_error.restype = C.c_char_p
    L.qd_launch_count.restype = c_ll
    for name in ("qd_qgemm_i8", "qd_quantize", "qd_groupnorm_quant", "qd_layernorm_quant", "qd_im2col_i8",
                 "qd_qattention", "qd_sampler_step", "qd_ancestral_step", "qd_split_bf16x3", "qd_attention_fp32",
                 "qd_embed_tokens", "qd_weight_scale_search"):
        getattr(L, name).argtypes = [c_vp, c_vp]
        getattr(L, name).restype = C.c_int
    L.qd_timestep_embedding.argtypes = [c_vp, c_vp, c_i32, c_i32, c_i32, c_vp, c_vp]
    L.qd_lincomb3.argtypes = [c_vp, c_f, c_vp, c_f, c_vp, c_f, c_vp, c_ll, c_vp]
    L.qd_copy2d.argtypes = [c_vp, c_ll, c_vp, c_ll, c_i32, c_i32, c_vp]
    L.qd_nchw_to_nhwc.argtypes = [c_vp, c_vp, c_i32, c_i32, c_i32, c_vp]
    L.qd_nhwc_to_nchw.argtypes = [c_vp, c_vp, c_i32, c_i32, c_i32, c_vp]
    L.qd_avgpool2x.argtypes = [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp]
    L.qd_upsample2x_f32.argtypes = [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp]
    L.qd_softmax_rows.argtypes = [c_vp, c_ll, c_i32, c_i32, c_vp]
    L.qd_vq_lookup.argtypes = [c_vp, c_ll, c_vp, c_vp, c_ll, c_i32, c_i32, c_i32, c_vp]
    L.qd_groupnorm_workspace_floats.argtypes = [c_i32, c_i32, c_i32, c_i32]
    L.qd_groupnorm_workspace_floats.restype = c_ll
    L.qd_engine_create.argtypes = [C.c_int, C.POINTER(c_vp)]
    L.qd_engine_add_op.argtypes = [c_vp, C.c_int, c_vp]
    L.qd_engine_num_ops.argtypes = [c_vp]
    L.qd_engine_finalize.argtypes = [c_vp]
    L.qd_engine_run.argtypes = [c_vp, c_vp]
    L.qd_engine_run_range.argtypes = [c_vp, C.c_int, C.c_int, c_vp]
    L.qd_engine_destroy.argtypes = [c_vp]
    L.qd_engine_destroy.restype = None
    _lib = L
    return L


def check(rc, what=""):
    if rc != 0:
        msg = lib().qd_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"qdiff_b200 {what} failed (status {rc}): {msg}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
