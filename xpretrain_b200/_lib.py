"""ctypes binding of the C-ABI library (include/xpretrain_b200.h).

There is deliberately no fallback: if `libxpretrain_b200.so` is missing, or a call is made without an
H100 (sm_90a), the error is raised to the caller.  Build with `python -c "import __graft_entry__ as g; g.build()"`
(or `make`) — the library is kept in-tree under xpretrain_b200/lib/.

The declarations below are a hand-written copy of the header, held to it by tests/test_boundary_cpu.py; `ops.py` is
their only caller.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libxpretrain_b200.so")

c_void_p, c_int, c_i64, c_float = C.c_void_p, C.c_int32, C.c_int64, C.c_float


class XpGemm(C.Structure):
    _fields_ = [
        ("a", c_void_p), ("b", c_void_p), ("c", c_void_p), ("bias", c_void_p), ("residual", c_void_p), ("aux", c_void_p),
        ("M", c_i64), ("N", c_i64), ("K", c_i64),
        ("lda", c_i64), ("ldb", c_i64), ("ldc", c_i64), ("ldr", c_i64), ("ld_aux", c_i64),
        ("a_layout", c_int), ("b_layout", c_int), ("act", c_int), ("out", c_int),
        ("splits", c_int), ("scale_cols", c_int), ("alpha", c_float), ("col_scale", c_float),
        ("c_group", c_i64), ("c_group_stride", c_i64), ("r_group", c_i64), ("r_group_stride", c_i64),
        ("block_n", c_int), ("max_ctas", c_int), ("cta_pair", c_int), ("reserved", c_int),
    ]


class XpRowMap(C.Structure):
    _fields_ = [("group", c_i64), ("group_stride", c_i64), ("ld", c_i64), ("offsets", c_void_p)]


class XpSegAttn(C.Structure):
    _fields_ = [("n_rows", c_i64), ("ld_qkv", c_i64), ("ld_out", c_i64), ("outer_stride", c_i64), ("inner_stride", c_i64),
                ("tok_stride", c_i64), ("heads", c_int), ("n_seq", c_int), ("seq_len", c_int), ("seg_len", c_int),
                ("inner", c_int), ("reserved", c_int), ("row_index", c_void_p), ("bias", c_void_p), ("ds_out", c_void_p),
                ("bias_windows", c_int), ("head_dim", c_int)]


class XpDenseAttn(C.Structure):
    _fields_ = [("n_rows", c_i64), ("ld_qkv", c_i64), ("ld_out", c_i64), ("heads", c_int), ("n_seq", c_int),
                ("seq_len", c_int), ("reserved", c_int)]


class XpNceGather(C.Structure):
    _fields_ = [("vis_local", c_void_p), ("txt_local", c_void_p), ("peer_bufs", c_void_p), ("logit_scale", c_void_p),
                ("g_scaled", c_void_p), ("vis_hi", c_void_p), ("txt_hi", c_void_p), ("loss", c_void_p),
                ("d_logit_scale", c_void_p), ("workspace", c_void_p), ("rank", c_int), ("world", c_int), ("b", c_int),
                ("d", c_int), ("epoch", C.c_uint32), ("mode", c_int), ("ld_g", c_i64)]


class XpNceTerm(C.Structure):
    _fields_ = [("axis", c_int), ("members", c_int), ("excl_diag", c_int), ("target", c_int)]


class XpNceTerms(C.Structure):
    _fields_ = [("z", c_void_p * 3), ("g", c_void_p * 3), ("ld", c_i64 * 3), ("n", c_int * 3), ("n_mats", c_int),
                ("n_terms", c_int), ("term", XpNceTerm * 6), ("logit_scale", c_void_p), ("scale", c_float),
                ("loss", c_void_p), ("d_logit_scale", c_void_p), ("workspace", c_void_p)]


# XpOptTensor as a numpy row type, filled column by column; `pb` (the column's earlier name) is a title: an alias
XpOptTensor = np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), (("pb", "p_bf16"), "<u8"), ("n", "<i8"),
                        ("step_size", "<f4"), ("decay", "<f4"), ("reserved", "<i4", (2,))])

ABI_VERSION = 1
ACT_NONE, ACT_QUICK_GELU, ACT_DQUICK_GELU, ACT_GELU_ERF, ACT_DGELU_ERF = 0, 1, 2, 3, 4
OUT_BF16, OUT_F32, OUT_F32_ATOMIC = 0, 1, 2
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2

P = C.POINTER
# name -> (restype, argtypes); every symbol include/xpretrain_b200.h declares
SIGNATURES = {
    "xp_version": (c_int, []),
    "xp_last_error": (C.c_char_p, []),
    "xp_launch_count": (c_i64, []),
    "xp_launch_count_reset": (None, []),
    "xp_gemm": (c_int, [P(XpGemm), c_void_p]),
    "xp_layernorm_fwd": (c_int, [c_void_p, P(XpRowMap), c_void_p, P(XpRowMap), c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_i64, c_int, c_float, c_void_p]),
    "xp_layernorm_add_fwd": (c_int, [c_void_p, P(XpRowMap), c_int, c_void_p, P(XpRowMap), c_void_p, P(XpRowMap), c_void_p,
                                     P(XpRowMap), c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_float,
                                     c_void_p]),
    "xp_layernorm_bwd": (c_int, [c_void_p, P(XpRowMap), c_void_p, P(XpRowMap), c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                 P(XpRowMap), c_void_p, P(XpRowMap), c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "xp_l2norm_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "xp_l2norm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "xp_frame_pool_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "xp_frame_pool_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_float, c_void_p]),
    "xp_lfvila_pool_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                   c_int, c_int, c_void_p]),
    "xp_lfvila_pool_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                   c_void_p]),
    "xp_lfvila_normalize_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "xp_lfvila_normalize_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "xp_lfvila_ce_fwd": (c_int, [c_void_p, c_i64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "xp_lfvila_ce_bwd": (c_int, [c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_int,
                                 c_int, c_void_p]),
    "xp_colsum_bf16": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_int, c_float, c_void_p]),
    "xp_cast_f32_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "xp_vip_patchify": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_int, c_int, c_int, c_void_p]),
    "xp_vip_patchify_u8": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_int, P(c_float), P(c_float), c_void_p]),
    "xp_vip_resize_patchify_u8": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_int, P(c_float), P(c_float),
                                          c_void_p]),
    "xp_lfvila_frames_patchify_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                             c_int, c_int, c_int, P(c_float), P(c_float), c_void_p]),
    "xp_vip_embed_tables": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                    c_int, c_int, c_int, c_void_p]),
    "xp_vip_embed_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_int, c_int, c_void_p]),
    "xp_text_embed_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                  c_void_p]),
    "xp_text_embed_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "xp_eos_offsets": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "xp_vip_attention_workspace_bytes": (c_i64, [c_int, c_int, c_int, c_int]),
    "xp_vip_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p]),
    "xp_vip_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                     c_int, c_int, c_int, c_float, c_void_p]),
    "xp_text_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "xp_text_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float,
                                      c_void_p]),
    "xp_nce_split": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "xp_nce_gather_exchange_bytes": (c_i64, [c_int, c_int, c_int]),
    "xp_nce_gather_workspace_bytes": (c_i64, [c_int]),
    "xp_nce_gather_fused": (c_int, [P(XpNceGather), c_void_p]),
    "xp_nce_terms_workspace_bytes": (c_i64, [P(XpNceTerms)]),
    "xp_nce_terms": (c_int, [P(XpNceTerms), c_void_p]),
    "xp_nce_dsl_workspace_bytes": (c_i64, [c_int]),
    "xp_nce_dsl": (c_int, [c_void_p, c_i64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "xp_seg_attention_fwd":(c_int, [c_void_p, c_void_p, c_void_p, P(XpSegAttn), c_void_p]),
    "xp_seg_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, P(XpSegAttn), c_float,
                                     c_void_p]),
    "xp_dense_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, P(XpDenseAttn), c_void_p]),
    "xp_dense_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, P(XpDenseAttn),
                                       c_float, c_void_p]),
    "xp_tsf_embed_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "xp_tsf_untokenize": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "xp_layernorm_wide_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_float,
                                      c_void_p]),
    "xp_layernorm_wide_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64,
                                      c_int, c_void_p]),
    "xp_gather_rows_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "xp_scatter_rows_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "xp_sim_f32":(c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_i64, c_void_p]),
    "xp_dsl_reweight": (c_int, [c_void_p, c_int, c_int, c_i64, c_float, c_void_p, c_void_p]),
    "xp_rank_counts": (c_int, [c_void_p, c_int, c_i64, c_int, c_void_p, c_void_p, c_void_p]),
    "xp_rowscale_bf16":(c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "xp_opt_chunk_elems": (c_int, []),
    "xp_opt_grad_norm": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p]),
    "xp_opt_scale_grads": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "xp_cast_table": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "xp_opt_adamw_step": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_float, c_float, c_float, c_void_p]),
}

_lib = None


class XpError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load the shared library once; raise loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise XpError(f"{LIB_PATH} not found: the CUDA extension is not built and there is no CPU fallback. "
                          f"Run `make` (or __graft_entry__.build()) in the repository root.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError here = header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise XpError(f"{what} failed: {lib().xp_last_error().decode()}")
