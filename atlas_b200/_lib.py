"""ctypes binding of the C-ABI library `lib/libatlas_b200.so` (declared in `include/atlas_b200.h`).

There is NO CPU fallback: if the library cannot be loaded, or a call is made without a CUDA
device, the functions here raise.  torch is used only for device memory and streams.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libatlas_b200.so")

OK = 0
MAX_TOPK = 1024
EMBEDDINGS_DIM = 768

_lib = None


class AtlasB200Error(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle; raise loudly if the CUDA library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AtlasB200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for this path)"
        )
    L = ctypes.CDLL(LIB_PATH)
    c = ctypes
    L.atlas_b200_last_error.restype = c.c_char_p
    L.atlas_b200_version.restype = c.c_char_p
    L.atlas_b200_launch_count.restype = c.c_uint64
    L.atlas_b200_mips_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_mips_workspace_bytes.argtypes = [c.c_int64, c.c_int32, c.c_int32]
    L.atlas_b200_mips_topk.restype = c.c_int
    L.atlas_b200_mips_topk.argtypes = [
        c.c_void_p, c.c_int64, c.c_int64, c.c_int32, c.c_void_p, c.c_int32, c.c_int32,
        c.c_void_p, c.c_void_p, c.c_int64, c.c_int64, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p,
    ]
    L.atlas_b200_mips_topk_exhaustive.restype = c.c_int
    L.atlas_b200_mips_topk_exhaustive.argtypes = [
        c.c_void_p, c.c_int64, c.c_int64, c.c_int32, c.c_void_p, c.c_int32, c.c_int32,
        c.c_void_p, c.c_void_p, c.c_int64, c.c_int64, c.c_void_p, c.c_size_t, c.c_void_p,
    ]
    L.atlas_b200_topk_merge.restype = c.c_int
    L.atlas_b200_topk_merge.argtypes = [
        c.c_void_p, c.c_void_p, c.c_int64, c.c_int64, c.c_int32, c.c_int32, c.c_int32, c.c_int32, c.c_int32,
        c.c_int32, c.c_void_p, c.c_void_p, c.c_void_p,
    ]
    L.atlas_b200_search_host.restype = c.c_int
    L.atlas_b200_search_host.argtypes = [
        c.c_void_p, c.c_int64, c.c_int64, c.c_int32, c.c_void_p, c.c_int32, c.c_int32,
        c.c_void_p, c.c_void_p, c.c_int64, c.c_int64, c.c_void_p, c.c_size_t, c.c_void_p,
    ]
    L.atlas_b200_cast_f32.restype = c.c_int
    L.atlas_b200_cast_f32.argtypes = [c.c_void_p, c.c_void_p, c.c_int64, c.c_int32, c.c_void_p]
    L.atlas_b200_linear_schedule.restype = c.c_int
    L.atlas_b200_linear_schedule.argtypes = [c.c_int32, c.c_int32, c.c_int32, c.c_int32]
    L.atlas_b200_layernorm.restype = c.c_int
    L.atlas_b200_layernorm.argtypes = [c.c_void_p, c.c_int64, c.c_void_p, c.c_void_p, c.c_void_p, c.c_int64, c.c_int32,
                                       c.c_int32, c.c_float, c.c_int32, c.c_int32, c.c_void_p]
    L.atlas_b200_bert_embed_ln.restype = c.c_int
    L.atlas_b200_bert_embed_ln.argtypes = [c.c_void_p] * 8 + [c.c_int32, c.c_int32, c.c_int32, c.c_float, c.c_int32,
                                                              c.c_void_p]
    L.atlas_b200_masked_mean_pool.restype = c.c_int
    L.atlas_b200_masked_mean_pool.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_int64, c.c_int32, c.c_int32,
                                              c.c_int32, c.c_int32, c.c_void_p]
    L.atlas_b200_profile_enable.restype = None
    L.atlas_b200_profile_enable.argtypes = [c.c_int32]
    L.atlas_b200_profile_work.restype = c.c_double
    L.atlas_b200_profile_work.argtypes = []
    L.atlas_b200_profile_launches.restype = c.c_int32
    L.atlas_b200_profile_launches.argtypes = [c.POINTER(c.c_double), c.POINTER(c.c_double), c.c_int32]
    L.atlas_b200_profile_collect.restype = c.c_int
    L.atlas_b200_profile_collect.argtypes = [c.POINTER(c.c_double), c.POINTER(c.c_int32)]
    i32, i64, vp, f32 = c.c_int32, c.c_int64, c.c_void_p, c.c_float
    L.atlas_b200_attention_combine_ex.restype = c.c_int
    L.atlas_b200_attention_combine_ex.argtypes = [vp, vp, i32, i32, i32, i32, vp, i64, vp, i32, vp]
    L.atlas_b200_cross_attention_stats.restype = c.c_int
    L.atlas_b200_cross_attention_stats.argtypes = [vp, i64, i32, vp, i64, i32, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32,
                                                   f32, i32, vp]
    L.atlas_b200_linear_wgrad.restype = c.c_int
    L.atlas_b200_linear_wgrad.argtypes = [vp, i64, vp, i64, vp, i64, i32, i32, i32, i32, vp, c.c_size_t, vp]
    L.atlas_b200_linear_wgrad_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_linear_wgrad_workspace_bytes.argtypes = [i32, i32, i32]
    L.atlas_b200_transpose.restype = c.c_int
    L.atlas_b200_transpose.argtypes = [vp, i64, vp, i64, i32, i32, i32, vp]
    L.atlas_b200_colsum.restype = c.c_int
    L.atlas_b200_colsum.argtypes = [vp, i64, vp, i32, i32, i32, vp]
    L.atlas_b200_layernorm_bwd.restype = c.c_int
    L.atlas_b200_layernorm_bwd.argtypes = [vp, i64, vp, i64, vp, vp, i64, vp, i64, vp, vp, i32, i32, f32, i32, i32, vp]
    L.atlas_b200_gated_gelu.restype = c.c_int
    L.atlas_b200_gated_gelu.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, i32, vp]
    L.atlas_b200_gelu_erf.restype = c.c_int
    L.atlas_b200_gelu_erf.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, i32, vp]
    L.atlas_b200_relu_bwd.restype = c.c_int
    L.atlas_b200_relu_bwd.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, i32, vp]
    L.atlas_b200_bert_embed_sum.restype = c.c_int
    L.atlas_b200_bert_embed_sum.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.atlas_b200_scatter_add_rows.restype = c.c_int
    L.atlas_b200_scatter_add_rows.argtypes = [vp, i32, vp, i64, vp, i64, i32, i64, i64, i32, vp]
    L.atlas_b200_masked_mean_pool_bwd.restype = c.c_int
    L.atlas_b200_masked_mean_pool_bwd.argtypes = [vp, i64, vp, vp, i32, i32, i32, i32, vp]
    L.atlas_b200_cross_entropy_fwd.restype = c.c_int
    L.atlas_b200_cross_entropy_fwd.argtypes = [vp, i64, vp, vp, vp, i32, i32, i32, vp]
    L.atlas_b200_cross_entropy_bwd.restype = c.c_int
    L.atlas_b200_cross_entropy_bwd.argtypes = [vp, i64, vp, vp, vp, vp, i64, i32, i32, i32, vp]
    L.atlas_b200_decode_cross_attention_live.restype = c.c_int
    L.atlas_b200_decode_cross_attention_live.argtypes = [vp, i64, vp, i64, i32, i32, vp, vp, i32, i32, i32, i32, f32, vp, vp, i32,
                                                         vp]
    L.atlas_b200_decode_self_attention.restype = c.c_int
    L.atlas_b200_decode_self_attention.argtypes = [vp, i64, vp, i32, vp, vp, f32, vp, i64, i32, i32, i32, vp]
    L.atlas_b200_decode_argmax.restype = c.c_int
    L.atlas_b200_decode_argmax.argtypes = [vp, i64, i32, vp, i64, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    L.atlas_b200_decode_self_attention_beam.restype = c.c_int
    L.atlas_b200_decode_self_attention_beam.argtypes = [vp, i64, vp, i32, vp, vp, vp, f32, vp, i64, i32, i32, i32, vp]
    L.atlas_b200_beam_topk.restype = c.c_int
    L.atlas_b200_beam_topk.argtypes = [vp, i64, i32, vp, i64, vp, vp, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp]
    L.atlas_b200_beam_select.restype = c.c_int
    L.atlas_b200_beam_select.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp,
                                         i32, i32, c.c_double, vp]
    L.atlas_b200_splice_tokens.restype = c.c_int
    L.atlas_b200_splice_tokens.argtypes = [vp, vp, i64, i64, vp, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp]
    u64 = c.c_uint64
    L.atlas_b200_dropout.restype = c.c_int
    L.atlas_b200_dropout.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, f32, u64, u64, vp, i32, vp]
    L.atlas_b200_dropout_mask.restype = c.c_int
    L.atlas_b200_dropout_mask.argtypes = [vp, i64, i32, f32, u64, u64, vp]
    L.atlas_b200_attention_train.restype = c.c_int
    L.atlas_b200_attention_train.argtypes = [vp, i64, i32, vp, i64, i32, vp, i64, i32, vp, i64, vp, vp, i32, i32, i32, i32,
                                             f32, f32, i32, vp, vp, vp, f32, u64, u64, vp, i32, vp]
    L.atlas_b200_attention_long.restype = c.c_int
    L.atlas_b200_attention_long.argtypes = [vp, i64, i32, vp, i64, i32, vp, i64, i32, vp, i64, vp, vp, i32, i32, i32, i32, f32,
                                            f32, vp, f32, u64, u64, vp, i32, vp]
    L.atlas_b200_attention_bwd_train.restype = c.c_int
    L.atlas_b200_attention_bwd_train.argtypes = [vp, i64, i32, vp, i64, i32, vp, i64, i32, vp, i64, vp, i64, vp, i64, i32,
                                                 vp, i64, i32, vp, i64, i32, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32,
                                                 f32, f32, f32, u64, u64, vp, i32, vp]
    L.atlas_b200_adamw_fp32copy.restype = c.c_int
    L.atlas_b200_adamw_fp32copy.argtypes = [vp, vp, i32, i32, f32, f32, f32, f32, f32, f32, vp]
    L.atlas_b200_grad_stats.restype = c.c_int
    L.atlas_b200_grad_stats.argtypes = [vp, i32, vp, i32, i32, vp, vp]
    L.atlas_b200_clamp_inf_fp16.restype = c.c_int
    L.atlas_b200_clamp_inf_fp16.argtypes = [vp, i64, i64, i32, vp, vp, vp, vp]
    L.atlas_b200_cross_attention_stream.restype = c.c_int
    L.atlas_b200_cross_attention_stream.argtypes = [vp, i64, i32, vp, i64, i32, i32, vp, vp, i32, i32, i32, i32, i32, f32, vp,
                                                    vp, i32, vp]
    L.atlas_b200_compact_live_tiles.restype = c.c_int
    L.atlas_b200_compact_live_tiles.argtypes = [vp, i64, vp, i32, i32, vp, i64, vp, vp, vp]
    L.atlas_b200_cross_attention_stream_compact.restype = c.c_int
    L.atlas_b200_cross_attention_stream_compact.argtypes = [vp, i64, i32, vp, i64, i32, i32, vp, vp, vp, i32, i32, i32, i32, i32,
                                                            f32, vp, vp, i32, vp]
    L.atlas_b200_attention_dropout_mask.restype = c.c_int
    L.atlas_b200_attention_dropout_mask.argtypes = [vp, i64, i32, f32, u64, u64, vp]
    L.atlas_b200_segment_tile_scan.restype = c.c_int
    L.atlas_b200_segment_tile_scan.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp]
    L.atlas_b200_embed_packed_tiles.restype = c.c_int
    L.atlas_b200_embed_packed_tiles.argtypes = [vp, vp, i64, i32, vp, i32, vp, i64, i32, vp]
    L.atlas_b200_linear_rows.restype = c.c_int
    L.atlas_b200_linear_rows.argtypes = [vp, i64, vp, i64, vp, vp, i64, vp, i64, i32, i32, i32, i32, i32, vp, vp, f32, vp, vp]
    L.atlas_b200_attention_packed.restype = c.c_int
    L.atlas_b200_attention_packed.argtypes = [vp, i64, i32, i32, i32, vp, i64, vp, vp, vp, vp, i32, i32, i32, f32, vp, f32, u64,
                                              u64, i32, vp]
    L.atlas_b200_attention_packed_bwd.restype = c.c_int
    L.atlas_b200_attention_packed_bwd.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32,
                                                  f32, f32, u64, u64, i32, vp]
    L.atlas_b200_expand_packed_tiles.restype = c.c_int
    L.atlas_b200_expand_packed_tiles.argtypes = [vp, i64, vp, i32, vp, i64, i32, vp]
    L.atlas_b200_quantize_kv_e4m3.restype = c.c_int
    L.atlas_b200_quantize_kv_e4m3.argtypes = [vp, i64, i64, i32, vp, i64, vp, i64, i32, vp]
    L.atlas_b200_decode_cross_attention_e4m3.restype = c.c_int
    L.atlas_b200_decode_cross_attention_e4m3.argtypes = [vp, i64, vp, i64, vp, i64, i32, i32, vp, vp, i32, i32, i32, i32, f32, vp,
                                                         vp, i32, vp]
    L.atlas_b200_cross_attention_stream_e4m3.restype = c.c_int
    L.atlas_b200_cross_attention_stream_e4m3.argtypes = [vp, i64, i32, vp, i64, vp, i64, i32, i32, vp, vp, i32, i32, i32, i32, i32,
                                                         f32, vp, vp, i32, vp]
    L.atlas_b200_pq_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_pq_workspace_bytes.argtypes = [i32, i64, i32, i32, i32]
    L.atlas_b200_pq_train.restype = c.c_int
    L.atlas_b200_pq_train.argtypes = [vp, i64, i32, i32, i32, vp, vp, vp, c.c_size_t, vp]
    L.atlas_b200_pq_encode.restype = c.c_int
    L.atlas_b200_pq_encode.argtypes = [vp, i64, i32, vp, vp, i32, vp, vp, vp, c.c_size_t, vp]
    L.atlas_b200_pq_topk.restype = c.c_int
    L.atlas_b200_pq_topk.argtypes = [vp, vp, i64, i32, vp, vp, i32, vp, i32, i32, vp, vp, i64, i64, vp, vp, c.c_size_t, vp]
    L.atlas_b200_pq_topk_exhaustive.restype = c.c_int
    L.atlas_b200_pq_topk_exhaustive.argtypes = [vp, vp, i64, i32, vp, vp, i32, vp, i32, i32, vp, vp, i64, i64, vp, c.c_size_t,
                                                vp]
    L.atlas_b200_pq_topk_probed.restype = c.c_int
    L.atlas_b200_pq_topk_probed.argtypes = [vp, vp, i64, i32, vp, vp, i32, vp, vp, i32, vp, i32, i32, vp, vp, i64, i64, vp, vp,
                                            c.c_size_t, vp]
    L.atlas_b200_pq_topk_probed_exhaustive.restype = c.c_int
    L.atlas_b200_pq_topk_probed_exhaustive.argtypes = [vp, vp, i64, i32, vp, vp, i32, vp, vp, i32, vp, i32, i32, vp, vp, i64,
                                                       i64, vp, c.c_size_t, vp]
    L.atlas_b200_ivfsq_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_ivfsq_workspace_bytes.argtypes = [i32, i64, i32, i32]
    L.atlas_b200_ivfsq_train.restype = c.c_int
    L.atlas_b200_ivfsq_train.argtypes = [vp, i64, i32, i32, vp, vp, vp, vp, c.c_size_t, vp]
    L.atlas_b200_ivfsq_encode.restype = c.c_int
    L.atlas_b200_ivfsq_encode.argtypes = [vp, i64, vp, i32, vp, vp, vp, vp, vp, vp, c.c_size_t, vp]
    L.atlas_b200_ivfsq_topk.restype = c.c_int
    L.atlas_b200_ivfsq_topk.argtypes = [vp, vp, vp, i64, i64, vp, i32, vp, vp, vp, i32, i32, vp, vp, i64, i64, vp, vp,
                                        c.c_size_t, vp]
    L.atlas_b200_ivfsq_topk_exhaustive.restype = c.c_int
    L.atlas_b200_ivfsq_topk_exhaustive.argtypes = [vp, vp, vp, i64, i64, vp, i32, vp, vp, vp, i32, i32, vp, vp, i64, i64, vp,
                                                   c.c_size_t, vp]
    L.atlas_b200_ivfsq_topk_probed.restype = c.c_int
    L.atlas_b200_ivfsq_topk_probed.argtypes = [vp, vp, vp, i64, i64, vp, vp, vp, i32, vp, vp, i32, vp, i32, i32, vp, vp, i64,
                                               i64, vp, vp, c.c_size_t, vp]
    L.atlas_b200_ivfsq_topk_probed_exhaustive.restype = c.c_int
    L.atlas_b200_ivfsq_topk_probed_exhaustive.argtypes = [vp, vp, vp, i64, i64, vp, vp, vp, i32, vp, vp, i32, vp, i32, i32,
                                                          vp, vp, i64, i64, vp, c.c_size_t, vp]
    L.atlas_b200_ivfflat_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_ivfflat_workspace_bytes.argtypes = [i32, i64, i32, i32]
    L.atlas_b200_ivfflat_topk.restype = c.c_int
    L.atlas_b200_ivfflat_topk.argtypes = [vp, vp, i64, i64, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, i64, i64, vp, vp,
                                          c.c_size_t, vp]
    L.atlas_b200_ivfflat_topk_exhaustive.restype = c.c_int
    L.atlas_b200_ivfflat_topk_exhaustive.argtypes = [vp, vp, i64, i64, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, i64, i64,
                                                     vp, c.c_size_t, vp]
    L.atlas_b200_pq_refine_workspace_bytes.restype = c.c_size_t
    L.atlas_b200_pq_refine_workspace_bytes.argtypes = [i32, i32]
    L.atlas_b200_pq_refine_topk.restype = c.c_int
    L.atlas_b200_pq_refine_topk.argtypes = [vp, i64, vp, i32, vp, i32, i32, vp, vp, i64, i64, vp, c.c_size_t, vp]
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "atlas_b200_last_error",
    "atlas_b200_version",
    "atlas_b200_launch_count",
    "atlas_b200_mips_workspace_bytes",
    "atlas_b200_mips_topk",
    "atlas_b200_mips_topk_exhaustive",
    "atlas_b200_topk_merge",
    "atlas_b200_search_host",
    "atlas_b200_cast_f32",
    "atlas_b200_linear_schedule",
    "atlas_b200_layernorm",
    "atlas_b200_bert_embed_ln",
    "atlas_b200_masked_mean_pool",
    "atlas_b200_profile_enable",
    "atlas_b200_profile_work",
    "atlas_b200_profile_collect",
    "atlas_b200_profile_launches",
    "atlas_b200_attention_combine_ex",
    "atlas_b200_cross_attention_stats",
    "atlas_b200_linear_wgrad",
    "atlas_b200_linear_wgrad_workspace_bytes",
    "atlas_b200_transpose",
    "atlas_b200_colsum",
    "atlas_b200_layernorm_bwd",
    "atlas_b200_gated_gelu",
    "atlas_b200_gelu_erf",
    "atlas_b200_relu_bwd",
    "atlas_b200_bert_embed_sum",
    "atlas_b200_scatter_add_rows",
    "atlas_b200_masked_mean_pool_bwd",
    "atlas_b200_cross_entropy_fwd",
    "atlas_b200_cross_entropy_bwd",
    "atlas_b200_splice_tokens",
    "atlas_b200_decode_self_attention",
    "atlas_b200_decode_argmax",
    "atlas_b200_decode_self_attention_beam",
    "atlas_b200_beam_topk",
    "atlas_b200_beam_select",
    "atlas_b200_dropout",
    "atlas_b200_dropout_mask",
    "atlas_b200_attention_dropout_mask",
    "atlas_b200_attention_train",
    "atlas_b200_attention_long",
    "atlas_b200_attention_bwd_train",
    "atlas_b200_adamw_fp32copy",
    "atlas_b200_grad_stats",
    "atlas_b200_clamp_inf_fp16",
    "atlas_b200_cross_attention_stream",
    "atlas_b200_decode_cross_attention_live",
    "atlas_b200_compact_live_tiles",
    "atlas_b200_cross_attention_stream_compact",
    "atlas_b200_segment_tile_scan",
    "atlas_b200_embed_packed_tiles",
    "atlas_b200_linear_rows",
    "atlas_b200_attention_packed",
    "atlas_b200_attention_packed_bwd",
    "atlas_b200_expand_packed_tiles",
    "atlas_b200_pq_workspace_bytes",
    "atlas_b200_pq_train",
    "atlas_b200_pq_encode",
    "atlas_b200_pq_topk",
    "atlas_b200_pq_topk_exhaustive",
    "atlas_b200_pq_topk_probed",
    "atlas_b200_pq_topk_probed_exhaustive",
    "atlas_b200_ivfsq_workspace_bytes",
    "atlas_b200_ivfsq_train",
    "atlas_b200_ivfsq_encode",
    "atlas_b200_ivfsq_topk",
    "atlas_b200_ivfsq_topk_exhaustive",
    "atlas_b200_ivfsq_topk_probed",
    "atlas_b200_ivfsq_topk_probed_exhaustive",
    "atlas_b200_ivfflat_workspace_bytes",
    "atlas_b200_ivfflat_topk",
    "atlas_b200_ivfflat_topk_exhaustive",
    "atlas_b200_pq_refine_workspace_bytes",
    "atlas_b200_pq_refine_topk",
    "atlas_b200_quantize_kv_e4m3",
    "atlas_b200_decode_cross_attention_e4m3",
    "atlas_b200_cross_attention_stream_e4m3",
]


def check(rc):
    if rc != OK:
        raise AtlasB200Error(f"atlas_b200 error {rc}: {lib().atlas_b200_last_error().decode()}")


def current_stream_ptr():
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(t, name):
    if not t.is_cuda:
        raise AtlasB200Error(f"{name} must be a CUDA tensor: atlas_b200 has no CPU path")
