"""ctypes binding of the C-ABI library (include/elliot_b200.h).

There is NO fallback: if the shared library is missing, or no CUDA device is present when a
compute entry point is called, an exception is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libelliot_b200.so")

c_i32, c_i64, c_u64, c_f32, c_f64 = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float, ctypes.c_double
c_int, c_void, c_size = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t

# name -> (restype, argtypes); mirrors include/elliot_b200.h one to one
SIGNATURES = {
    "eb_last_error": (ctypes.c_char_p, []),
    "eb_version": (c_int, []),
    "eb_device_info": (c_int, [c_void, c_void]),
    "eb_bpr_step_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_void, c_void, c_void, c_i64,
                                c_f32, c_f32, c_f32, c_f32, c_f32, c_void, c_int, c_void]),
    "eb_bpr_step_sampled_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_i32, c_i32, c_void, c_void,
                                        c_i64, c_u64, c_u64, c_f32, c_f32, c_f32, c_f32, c_f32,
                                        c_void, c_void, c_void, c_void, c_void, c_size, c_int, c_void]),
    "eb_bpr_step_sampled_workspace_bytes": (c_size, [c_i64, c_i32]),
    "eb_bloom_build": (c_int, [c_void, c_void, c_i32, c_int, c_void, c_void]),
    "eb_bpr_step_sampled_filter_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_i32, c_i32, c_void, c_void, c_void, c_int,
                                               c_i64, c_u64, c_u64, c_f32, c_f32, c_f32, c_f32, c_f32,
                                               c_void, c_void, c_void, c_void, c_void, c_size, c_int, c_void]),
    "eb_bpr_schedule_sampled": (c_int, [c_i32, c_i32, c_void, c_i64, c_u64, c_u64, c_void, c_size, ctypes.POINTER(c_size), c_int,
                                        c_void]),
    "eb_bpr_apply_sampled_filter_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_i32, c_i32, c_void, c_void, c_void, c_int,
                                                c_i64, c_u64, c_u64, c_f32, c_f32, c_f32, c_f32, c_f32,
                                                c_void, c_void, c_void, c_void, c_void, c_int, c_void]),
    "eb_bpr_sample_philox_filter": (c_int, [c_i32, c_i32, c_void, c_void, c_void, c_int, c_i64, c_u64, c_u64, c_void, c_void, c_void,
                                            c_void]),
    "eb_bpr_sample_philox": (c_int, [c_i32, c_i32, c_void, c_void, c_i64, c_u64, c_u64, c_void, c_void, c_void,
                                     c_void]),
    "eb_bpr_step_host_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_void, c_void, c_void, c_i64,
                                     c_f32, c_f32, c_f32, c_f32, c_f32, c_void, c_void, c_void, c_int, c_void]),
    "eb_bpr_step_host_packed_f32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_void, c_i64, c_int, c_int,
                                            c_f32, c_f32, c_f32, c_f32, c_f32, c_void, c_void, c_void, c_int, c_void]),
    "eb_bpr_exact_workspace_bytes": (c_size, [c_i64, c_i32, c_i32]),
    "eb_bpr_exact_f64": (c_int, [c_void, c_void, c_void, c_int, c_int, c_i32, c_i32, c_void, c_void, c_void, c_i64,
                                 c_f64, c_f64, c_f64, c_f64, c_f64, c_void, c_void, c_size, c_void]),
    "eb_mt_seed": (c_int, [c_void, ctypes.c_uint32, c_void]),
    "eb_mt_sampler_workspace_bytes": (c_size, [c_i64]),
    "eb_mt_sampler_step": (c_int, [c_void, c_i32, c_i32, c_void, c_void, c_void, c_i64, c_void, c_void, c_void,
                                   c_void, c_size, c_void]),
    "eb_mt_raw": (c_int, [c_void, c_void, c_i64, c_void]),
    "eb_score_topk_workspace_bytes": (c_size, [c_i64, c_i32, c_int]),
    "eb_score_topk_f32": (c_int, [c_void, c_void, c_void, c_i32, c_int, c_int, c_void, c_void, c_void, c_i32, c_i64,
                                  c_int, c_void, c_void, c_void, c_size, c_void]),
    "eb_score_topk_f64": (c_int, [c_void, c_void, c_void, c_i32, c_int, c_int, c_void, c_void, c_void, c_i32, c_i64,
                                  c_int, c_void, c_void, c_void, c_size, c_void]),
    "eb_bpr_batch_grad_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_void, c_int, c_int, c_void, c_void, c_void,
                                      c_i64, c_f32, c_f32, c_void, c_void]),
    "eb_adam_dense_f32": (c_int, [c_void, c_void, c_void, c_void, c_i64, c_f32, c_f32, c_f32, c_f32, c_i64, c_void]),
    "eb_adam_dense_copy_f32": (c_int, [c_void, c_void, c_void, c_void, c_i64, c_f32, c_f32, c_f32, c_f32, c_i64, c_void, c_void]),
    "eb_convert_bf16": (c_int, [c_void, c_int, c_int, c_i64, c_void, c_i64, c_int, c_void]),
    "eb_gemm_bf16_tn": (c_int, [c_void, c_i64, c_void, c_i64, c_void, c_i64, c_int, c_int, c_int, c_void, c_f32, c_int,
                                c_void]),
    "eb_gemm_bf16": (c_int, [c_void, c_i64, c_int, c_void, c_i64, c_int, c_void, c_i64, c_int, c_int, c_int, c_void, c_f32, c_int,
                             c_void]),
    "eb_gemm_bf16_out": (c_int, [c_void, c_i64, c_int, c_void, c_i64, c_int, c_void, c_i64, c_void, c_i64, c_int, c_int, c_int, c_void,
                                 c_f32, c_int, c_void]),
    "eb_gemm_f32_ref": (c_int, [c_void, c_i64, c_int, c_void, c_i64, c_int, c_void, c_i64, c_int, c_int, c_int, c_void, c_f32, c_int,
                                c_void]),
    "eb_vae_embed_fwd": (c_int, [c_void, c_void, c_int, c_void, c_void, c_void, c_int, c_void, c_i64, c_f32, c_u64, c_void]),
    "eb_vae_embed_bwd": (c_int, [c_void, c_int, c_void, c_void, c_void, c_int, c_void, c_i64, c_f32, c_u64, c_void]),
    "eb_vae_reparam_fwd": (c_int, [c_void, c_i64, c_int, c_int, c_void, c_i64, c_u64, c_u64, c_void, c_void]),
    "eb_vae_reparam_bwd": (c_int, [c_void, c_i64, c_int, c_int, c_void, c_i64, c_void, c_i64, c_u64, c_u64, c_f32, c_void]),
    "eb_vae_softmax": (c_int, [c_void, c_i64, c_int, c_void, c_void, c_void, c_int, c_void, c_void, c_int, c_void]),
    "eb_vae_softmax_bf16": (c_int, [c_void, c_i64, c_int, c_void, c_void, c_void, c_int, c_void, c_void, c_int, c_void, c_i64, c_void]),
    "eb_tanh_bwd": (c_int, [c_void, c_void, c_void, c_i64, c_void]),
    "eb_colsum": (c_int, [c_void, c_int, c_int, c_i64, c_void, c_void]),
    "eb_dense_topk_f32": (c_int, [c_void, c_i64, c_int, c_int, c_void, c_void, c_void, c_void, c_int, c_void, c_void, c_void]),
    "eb_neumf_gather": (c_int, [c_void, c_void, c_void, c_void, c_int, c_i64, c_void, c_void, c_i64, c_void, c_i64, c_void, c_i64, c_void]),
    "eb_neumf_head": (c_int, [c_void, c_i64, c_void, c_i64, c_int, c_void, c_void, c_void, c_i64, c_void, c_void, c_void, c_void,
                              c_void, c_void, c_void]),
    "eb_neumf_head_norm": (c_int, [c_void, c_i64, c_void, c_i64, c_int, c_void, c_void, c_void, c_i64, c_i64, c_void, c_void, c_void,
                                   c_void, c_void, c_void, c_void]),
    "eb_relu_bwd_copy": (c_int, [c_void, c_void, c_void, c_i64, c_void, c_void]),
    "eb_relu_bwd": (c_int, [c_void, c_void, c_void, c_i64, c_void]),
    "eb_neumf_scatter": (c_int, [c_void, c_void, c_int, c_i64, c_void, c_void, c_i64, c_void, c_i64, c_void, c_i64, c_void, c_void,
                                 c_void, c_void, c_void]),
    "eb_neumf_sample": (c_int, [c_i32, c_i32, c_void, c_void, c_int, c_u64, c_i64, c_void, c_void, c_void, c_void]),
    "eb_neumf_pair_h1": (c_int, [c_void, c_i64, c_void, c_i64, c_void, c_int, c_int, c_int, c_void, c_i64, c_void]),
    "eb_neumf_pair_h1_f32": (c_int, [c_void, c_i64, c_void, c_i64, c_void, c_int, c_int, c_int, c_void, c_i64, c_void]),
    "eb_neumf_pair_head": (c_int, [c_void, c_void, c_i64, c_int, c_int, c_int, c_int, c_void, c_i64, c_void, c_void, c_void, c_i64,
                                   c_void]),
    "eb_gather_rows_f32": (c_int, [c_void, c_i64, c_void, c_i64, c_int, c_void, c_i64, c_void]),
    "eb_scatter_add_rows_f32": (c_int, [c_void, c_i64, c_void, c_i64, c_int, c_void, c_i64, c_void]),
    "eb_bpr_step_rows_f32": (c_int, [c_void, c_i64, c_void, c_void, c_void, c_i64, c_i64, c_int, c_f32, c_f32, c_f32, c_f32, c_f32,
                                     c_void, c_void, c_void, c_void]),
    "eb_table_delta_f32": (c_int, [c_void, c_void, c_void, c_i64, c_void]),
    "eb_table_apply_delta_f32": (c_int, [c_void, c_void, c_void, c_i64, c_f32, c_void]),
    "eb_vae_step_workspace_bytes": (c_size, [c_int, c_int, c_int, c_int]),
    "eb_vae_train_step": (c_int, [c_void, c_void, c_int, c_f32, c_u64, c_u64, c_u64, c_f32, c_f32, c_void, c_void, c_size, c_int, c_void]),
    "eb_mf_pointwise_exact_f64": (c_int, [c_void, c_void, c_void, c_void, c_void, c_int, c_int, c_void, c_void, c_void, c_i64,
                                  c_f64, c_f64, c_i64, c_void, c_void]),
    "eb_mf_pointwise_step_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_int, c_int, c_void, c_void, c_i64, c_int, c_i32,
                                 c_u64, c_u64, c_i64, c_i64, c_f32, c_f32, c_void, c_void, c_void, c_void, c_void, c_void]),
    "eb_eval_topk_workspace_bytes": (c_size, [c_i64, c_int]),
    "eb_eval_topk_f64": (c_int, [c_void, c_i64, c_int, c_int, c_void, c_void, c_void, c_void, c_void, c_void, c_void, c_void,
                         c_void, c_size, c_void]),
    "eb_partition_streams_create": (c_int, [c_int, c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(c_int)]),
    "eb_table_apply_delta_late_f32": (c_int, [c_void, c_void, c_void, c_void, c_i64, c_f32, c_void]),
    "eb_gmf_step_grads": (c_int, [c_void, c_void, c_i64, c_int, c_void, c_void, c_void, c_void, c_i64, c_i64, c_void, c_void, c_void,
                                  c_void, c_void]),
    "eb_gmf_scale_rows": (c_int, [c_void, c_i64, c_i64, c_int, c_void, c_void, c_i64, c_void]),
    "eb_sigmoid_inplace": (c_int, [c_void, c_i64, c_void]),
    "eb_pointwise_sample_philox": (c_int, [c_i32, c_i32, c_void, c_void, c_void, c_int, c_i64, c_u64, c_u64, c_void, c_void, c_void,
                                           c_void]),
    "eb_peer_alloc": (c_int, [c_size, ctypes.POINTER(ctypes.c_void_p)]),
    "eb_peer_free": (c_int, [c_void]),
    "eb_peer_export": (c_int, [c_void, c_void]),
    "eb_peer_open": (c_int, [c_void, ctypes.POINTER(ctypes.c_void_p)]),
    "eb_peer_close": (c_int, [c_void]),
    "eb_bpr_step_peer_f32": (c_int, [c_void, c_void, c_void, c_int, c_i32, c_int, c_int, c_i32, c_void, c_void, c_void, c_i64,
                                     c_f32, c_f32, c_f32, c_f32, c_f32, c_void, c_int, c_void]),
    "eb_bpr_step_sampled_peer_f32": (c_int, [c_void, c_void, c_void, c_int, c_i32, c_int, c_int, c_i32, c_i32, c_void, c_void,
                                             c_void, c_int, c_i64, c_u64, c_u64, c_f32, c_f32, c_f32, c_f32, c_f32, c_void, c_void, c_void,
                                             c_void, c_int, c_void]),
    "eb_table_reconcile_peer_f32": (c_int, [c_void, c_int, c_void, c_i64, c_f32, c_int, c_void]),
    "eb_neumf_gather_peer": (c_int, [c_void, c_void, c_i64, c_void, c_int, c_i32, c_i64, c_int, c_void, c_void, c_i64, c_void,
                                     c_i64, c_void, c_i64, c_void]),
    "eb_neumf_scatter_peer": (c_int, [c_void, c_i64, c_void, c_void, c_int, c_i32, c_i64, c_int, c_void, c_void, c_i64, c_void,
                                      c_i64, c_void, c_i64, c_void, c_void, c_void]),
    "eb_group_by_owner_i32": (c_int, [c_void, c_void, c_void, c_int, c_int, c_i64, c_i32, c_int, c_int, c_void, c_void, c_void, c_void,
                                      c_void]),
    "eb_gather_rows_peer_f32": (c_int, [c_void, c_int, c_i32, c_i64, c_void, c_i64, c_int, c_void, c_i64, c_void]),
    "eb_score_topk_tc_workspace_bytes": (c_size, [c_i64, c_i32, c_int]),
    "eb_score_topk_tc_f32": (c_int, [c_void, c_void, c_void, c_i32, c_int, c_int, c_void, c_void, c_i32, c_i64, c_int,
                                     c_void, c_void, c_void, c_void, c_size, c_void, c_void]),
    "eb_csr_to_dense_bf16": (c_int, [c_void, c_void, c_void, c_i32, c_i32, c_i32, c_f32, c_void, c_i64, c_void, c_void, c_void]),
    "eb_knn_neighbors_f32": (c_int, [c_void, c_i64, c_i32, c_i32, c_i32, c_void, c_int, c_f32, c_int, c_void, c_void, c_void,
                                     c_void]),
    "eb_knn_score_tile_cols": (c_int, []),
    "eb_knn_score_topk_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_void, c_i32, c_void, c_void, c_void, c_i32, c_i64,
                                      c_int, c_int, c_void, c_void, c_void]),
    "eb_gram_f64_workspace_bytes": (c_size, [c_i64, c_int]),
    "eb_gram_f64": (c_int, [c_void, c_i64, c_int, c_i64, c_void, c_void, c_size, c_void]),
    "eb_als_small_d_max": (c_int, []),
    "eb_als_solve_f64": (c_int, [c_void, c_void, c_i64, c_int, c_void, c_void, c_void, c_void, c_void, c_i64, c_f64, c_void, c_i64,
                                 c_void]),
    "eb_inverse_f64_workspace_bytes": (c_size, [c_i64]),
    "eb_inverse_f64": (c_int, [c_void, c_i64, c_i64, c_void, c_size, c_void]),
    "eb_ease_normal_f64": (c_int, [c_void, c_i64, c_i32, c_i64, c_i64, c_void, c_f64, c_f64, c_void, c_i64, c_void]),
    "eb_ease_weights_f32": (c_int, [c_void, c_i64, c_i64, c_void, c_i64, c_void]),
    "eb_dense_score_topk_f32": (c_int, [c_void, c_void, c_void, c_void, c_i64, c_i32, c_void, c_void, c_void, c_i32, c_i64,
                                        c_int, c_int, c_void, c_void, c_void]),
    "eb_rp3_tile_cols": (c_int, []),
    "eb_rp3_row_workspace_bytes": (c_size, [c_i32]),
    "eb_rp3_similarity_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_void, c_void, c_i32, c_void, c_int, c_i64,
                                      c_void, c_void, c_void, c_void, c_size, c_void]),
    "eb_rp3_l1_rows_f32": (c_int, [c_i32, c_i64, c_void, c_void, c_void]),
    "eb_rp3_prune_workspace_bytes": (c_size, [c_i32, c_i64, c_i64]),
    "eb_rp3_prune_cols_f32": (c_int, [c_i32, c_i64, c_void, c_void, c_void, c_i64, c_int, c_void, c_void, c_void, c_void, c_size,
                                      c_void]),
    "eb_rp3_score_topk_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_void, c_i32, c_void, c_void, c_void, c_i32, c_i64,
                                      c_void, c_int, c_void, c_void, c_void, c_size, c_void]),
    "eb_slim_shared_residual_fits": (c_int, [c_i32]),
    "eb_slim_slots": (c_int, [c_i32, c_int]),
    "eb_slim_workspace_bytes": (c_size, [c_i32, c_i32, c_i32, c_int]),
    "eb_slim_fit_f32": (c_int, [c_void, c_void, c_void, c_void, c_void, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, c_f32,
                                ctypes.c_uint32, c_int, c_int, c_int, c_i32, c_void, c_void, c_void, c_void, c_void, c_void,
                                c_size, c_void]),
    "eb_slim_drop_f32": (c_int, [c_i32, c_void, c_void, c_void]),
    "eb_svd_max_width": (c_int, []),
    "eb_csr_spmm_f64": (c_int, [c_void, c_void, c_void, c_i64, c_void, c_int, c_i64, c_void, c_i64, c_void]),
    "eb_chol_pivoted_f64": (c_int, [c_void, c_int, c_void, c_void, c_void]),
    "eb_tall_times_small_f64": (c_int, [c_void, c_i64, c_int, c_i64, c_void, c_int, c_void, c_i64, c_void]),
    "eb_sym_eig_f64_workspace_bytes": (c_size, [c_int]),
    "eb_sym_eig_f64": (c_int, [c_void, c_int, c_void, c_void, c_void, c_size, c_void]),
    "eb_svd_finish_f64": (c_int, [c_void, c_int, c_int, c_void, c_i64, c_i64, c_void, c_i64, c_i64, c_int, c_void, c_void]),
    "eb_slope_one_dev_f64": (c_int, [c_void, c_void, c_void, c_i64, c_i32, c_i32, c_int, c_void, c_i64, c_void]),
    "eb_slope_one_score_topk_f64": (c_int, [c_void, c_i64, c_i32, c_void, c_void, c_void, c_void, c_void, c_void, c_i32, c_i64,
                                            c_int, c_void, c_void, c_void]),
    "eb_nnmf_dots_f64": (c_int, [c_void, c_void, c_int, c_void, c_void, c_i32, c_void, c_void]),
    "eb_nnmf_bias_chain_f64": (c_int, [c_void, c_void, c_void, c_void, c_i32, c_i32, c_f64, c_f64, c_f64, c_void, c_void,
                                       c_void, c_void]),
    "eb_nnmf_row_update_f64": (c_int, [c_void, c_void, c_void, c_i32, c_void, c_void, c_void, c_void, c_void, c_int, c_f64,
                                       c_void]),
}

_lib = None


class EbError(RuntimeError):
    pass


def lib():
    """Load libelliot_b200.so (built by `python -m elliot_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EbError(f"{LIB_PATH} is missing: build it with `python -m elliot_b200.build` "
                          f"(there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        msg = lib().eb_last_error().decode("utf-8", "replace")
        raise EbError(f"elliot_b200 C-ABI error {rc}: {msg}")
