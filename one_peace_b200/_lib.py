"""ctypes loader for ``csrc/libonepeace_b200.so`` (the C-ABI declared in ``include/onepeace_b200.h``).

The product path has no CPU or PyTorch fallback: if the shared library is missing the import of this
module raises, and every non-zero status from a C entry point raises ``RuntimeError`` (the reference's
error convention is Python exceptions only, SURVEY.md §8b).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OPB_LIB_PATH") or os.path.join(_HERE, "csrc", "libonepeace_b200.so")   # override: instrumented builds

c_void_p, c_int, c_int64, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

# name -> (restype, argtypes); must list every symbol include/onepeace_b200.h declares
# (tests/test_abi_symbols.py cross-checks this table against the header).
SIGNATURES = {
    "opb_abi_version": (c_int, []),
    "opb_status_string": (ctypes.c_char_p, [c_int]),
    "opb_gemm_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_int64,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int,
                              c_int, c_int, c_void_p]),
    "opb_grouped_conv1d_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int64,
                                        c_void_p, c_void_p]),
    "opb_pack_group_halo": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_int, c_void_p]),
    "opb_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_int64, c_void_p]),
    "opb_attention_tc_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_relpos_lut_build": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_relpos_decomp_proj": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int,
                                       c_int, c_int, c_int, c_int, c_void_p]),
    "opb_attention_decomp_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "opb_attention_temporal_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_attention_temporal_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float,
                                           c_void_p]),
    "opb_ms_deform_attn_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "opb_ms_deform_attn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "opb_seg_dwconv_gelu": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "opb_seg_out_map": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_gemm_bf16_ex": (c_int, [c_void_p, c_void_p]),
    "opb_row_stats_cast": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "opb_ln_stats_finalize": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "opb_layernorm": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int, c_int,
                              c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_text_embed": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_int, c_void_p]),
    "opb_image_patchify4": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "opb_cls_row_init": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "opb_relpos_bias_build": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "opb_audio_frame10": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int64, c_void_p]),
    "opb_l2_normalize_rows": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_zero_padded_rows": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_transpose_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p]),
    "opb_split_bf16x3": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_infonce_ws_floats": (c_int64, [c_int, c_int]),
    "opb_infonce_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                 c_float, c_void_p, c_void_p, c_void_p, c_int, c_float, c_void_p]),
    "opb_infonce_dscale": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "opb_infonce_lse_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "opb_infonce_merge_reduce": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p]),
    "opb_adam_chunk_elems": (c_int, []),
    "opb_adam_multi_step": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_float,
                                    c_float, c_float, c_void_p, c_void_p]),
    "opb_grad_norm_clip": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_float, c_float, c_void_p, c_void_p]),
    "opb_adan_multi_step": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int, c_float, c_float, c_float, c_float, c_void_p, c_void_p]),
}

SIGNATURES.update({
    "opb_bwd_ws_floats": (c_int64, [c_int]),
    "opb_layernorm_bwd": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int64, c_int, c_int, c_int, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                  c_void_p]),
    "opb_topk10_rows": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_recall_hits": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "opb_window_gather": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_window_scatter": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_batch_sum_f32": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "opb_l2_normalize_bwd": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_text_embed_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "opb_geglu_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "opb_geglu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "opb_gelu_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "opb_gelu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "opb_scale_resid_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "opb_scale_resid_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                    c_int, c_int, c_int, c_int, c_void_p]),
    "opb_colsum_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "opb_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_int, c_int, c_int, c_int, c_float, c_int64, c_void_p]),
    "opb_row_gather": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int, c_int64,
                               c_int64, c_int, c_void_p]),
    "opb_row_scatter_add": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p]),
    "opb_relpos_bias_block": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int,
                                      c_int, c_int, c_void_p]),
    "opb_relpos_bias_block_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int,
                                          c_int, c_int, c_void_p]),
    "opb_relpos_bias_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "opb_attention_bwd_t": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int, c_int, c_int, c_float, c_void_p]),
    "opb_relpos_bias_transpose": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "opb_relpos_dbias_fold": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "opb_relpos_dbias_center": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p]),
    "opb_gemm_bf16_t": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int64,
                                c_void_p, c_int, c_void_p]),
    "opb_ln_fold": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int64,
                            c_void_p, c_void_p, c_void_p]),
    "opb_attn_pool_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "opb_attn_pool_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                  c_int, c_void_p]),
    "opb_classify_loss": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_float, c_int, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "opb_refcoco_loss": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "opb_iou_acc": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "opb_argmax_hits": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                                c_void_p]),
    "opb_sum_f64": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "opb_sigmoid_pack": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64,
                                 c_void_p, c_void_p]),
    "opb_average_precision_ws_bytes": (c_int64, [c_int, c_int]),
    "opb_average_precision": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    "opb_token_mean_ln_ws_floats": (c_int64, [c_int, c_int, c_int]),
    "opb_token_mean_ln_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int64,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "opb_token_mean_ln_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_int64, c_void_p]),
})


class GemmArgs(ctypes.Structure):
    """Mirror of `opb_gemm_args` (include/onepeace_b200.h)."""
    _fields_ = [("A", c_void_p), ("lda", c_int64), ("B", c_void_p), ("ldb", c_int64),
                ("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32), ("epi", ctypes.c_int32),
                ("out", c_void_p), ("ldo", c_int64),
                ("bias", c_void_p), ("colscale", c_void_p), ("gamma", c_void_p), ("resid", c_void_p), ("ldr", c_int64),
                ("out_group", ctypes.c_int32), ("out_group_stride", ctypes.c_int32), ("out_row_offset", ctypes.c_int32),
                ("out_group_valid", ctypes.c_int32), ("resid_period", ctypes.c_int32), ("resid_row_offset", ctypes.c_int32),
                ("ln_mu", c_void_p), ("ln_rstd", c_void_p), ("ln_colsum", c_void_p),
                ("stats_out", c_void_p), ("out_bf16", c_void_p), ("ldo_bf16", c_int64),
                ("cta_group", ctypes.c_int32), ("reserved", ctypes.c_int32),
                ("workspace", c_void_p), ("workspace_bytes", c_int64),
                ("ln_partial", c_void_p), ("ln_parts", ctypes.c_int32), ("ln_dim", ctypes.c_int32), ("ln_eps", c_float),
                ("reserved2", ctypes.c_int32)]


_lib = None


def build_hint():
    return ("build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C one_peace_b200/csrc`")


def load():
    """Load the shared library once; raise if it is absent (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: the sm_90a extension is required; {build_hint()}")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so is stale
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().opb_status_string(status).decode()
        raise RuntimeError(f"{what}: {msg} (status {status})")
