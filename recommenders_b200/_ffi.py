"""ctypes binding of libtfrs_b200.so (the C ABI declared in include/tfrs_b200.h).

There is NO CPU fallback: if the library is missing or a tensor is not on a CUDA device the call
fails loudly.  PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TFRS_B200_LIB", os.path.join(_HERE, "libtfrs_b200.so"))

_lib: Optional[ctypes.CDLL] = None

I32, I64, BYTES = 0, 1, 2
F32, F64, BOOL = 3, 4, 5
c_p = ctypes.c_void_p
c_i = ctypes.c_int
c_l = ctypes.c_int64
c_f = ctypes.c_float
c_sz = ctypes.c_size_t
c_u32 = ctypes.c_uint32
c_u64 = ctypes.c_uint64
c_d = ctypes.c_double

_SIGNATURES = {
    "tfrs_version": (c_i, []),
    "tfrs_last_error": (ctypes.c_char_p, []),
    "tfrs_launch_count": (c_l, []),
    "tfrs_gather_f32": (c_i, [c_p, c_p, c_p, c_i, c_p, c_i, c_l, c_p, c_l, c_p, c_p]),
    "tfrs_topk_scan_workspace_bytes": (c_sz, [c_l, c_l, c_i, c_i]),
    "tfrs_topk_scan_f32": (c_i, [c_p, c_l, c_p, c_l, c_i, c_i, c_l, c_p, c_p, c_i, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_index_bytes": (c_sz, [c_l, c_i]),
    "tfrs_index_build": (c_i, [c_p, c_l, c_i, c_p, c_sz, c_p]),
    "tfrs_topk_tc_workspace_bytes": (c_sz, [c_l, c_l, c_i, c_i]),
    "tfrs_topk_tc_f32": (c_i, [c_p, c_l, c_p, c_p, c_l, c_i, c_i, c_l, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_topk_tc_exclude_f32": (c_i, [c_p, c_l, c_p, c_p, c_l, c_i, c_i, c_l, c_p, c_p, c_i, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_topk_tc_count_f32": (c_i, [c_p, c_l, c_p, c_p, c_l, c_i, c_i, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_topk_exclude_rerank_f32": (c_i, [c_p, c_p, c_l, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p]),
    "tfrs_count_above_f32": (c_i, [c_p, c_l, c_i, c_p, c_l, c_p, c_p]),
    "tfrs_topk_hits_accumulate": (c_i, [c_p, c_p, c_p, c_l, c_p, c_i, c_p, c_p]),
    "tfrs_topk_tc_layout": (c_i, [c_l, c_l, c_i, c_i, c_p]),
    "tfrs_topk_tc_retry_layout": (c_i, [c_l, c_l, c_i, c_i, c_p]),
    "tfrs_topk_tc_sample_layout": (c_i, [c_l, c_l, c_i, c_i, c_p]),
    "tfrs_dot_interaction_out_dim": (c_i, [c_i, c_i, c_i]),
    "tfrs_dot_interaction_fwd_f32": (c_i, [c_p, c_l, c_i, c_i, c_i, c_i, c_p, c_p]),
    "tfrs_dot_interaction_bwd_f32": (c_i, [c_p, c_p, c_l, c_i, c_i, c_i, c_i, c_p, c_p]),
    "tfrs_profile_enable": (c_i, [c_i]),
    "tfrs_profile_read": (c_i, [c_p, c_p]),
    "tfrs_topk_merge_strided": (c_i, [c_p, c_p, c_l, c_l, c_i, c_l, c_i, c_i, c_p, c_p, c_p]),
    "tfrs_topk_merge_sorted_strided": (c_i, [c_p, c_p, c_l, c_l, c_i, c_l, c_i, c_i, c_p, c_p, c_p]),
    "tfrs_topk_override_merge_f32": (c_i, [c_p, c_p, c_l, c_i, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i, c_p]),
    "tfrs_topk_overriding_dense_workspace_bytes": (c_sz, [c_l, c_l, c_i, c_i]),
    "tfrs_topk_overriding_dense_f32": (c_i, [c_p, c_p, c_l, c_p, c_l, c_i, c_i, c_p, c_p, c_p, c_p, c_i, c_p, c_sz, c_p]),
    "tfrs_count_listed": (c_i, [c_p, c_l, c_i, c_l, c_p, c_p, c_p, c_p]),
    "tfrs_comm_unique_id": (c_i, [c_p]),
    "tfrs_comm_create": (c_i, [c_p, c_i, c_i, c_p]),
    "tfrs_comm_destroy": (c_i, [c_p]),
    "tfrs_comm_enable_p2p": (c_i, [c_p, c_l, c_i]),
    "tfrs_comm_p2p_capacity": (c_i, [c_p, c_l, c_i]),
    "tfrs_comm_set_option": (c_i, [c_p, c_i, c_i]),
    "tfrs_comm_rank": (c_i, [c_p]),
    "tfrs_comm_world": (c_i, [c_p]),
    "tfrs_topk_allgather": (c_i, [c_p, c_p, c_p, c_l, c_i, c_p, c_p, c_p]),
    "tfrs_topk_sharded_workspace_bytes": (c_sz, [c_i, c_l, c_l, c_i, c_i]),
    "tfrs_topk_sharded_layout": (c_i, [c_i, c_l, c_l, c_i, c_i, c_p]),
    "tfrs_topk_sharded_f32": (c_i, [c_p, c_p, c_l, c_p, c_p, c_l, c_i, c_i, c_l, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_sgemm_f32": (c_i, [c_i, c_i, c_l, c_l, c_l, c_p, c_l, c_p, c_l, c_p, c_l, c_i, c_p]),
    "tfrs_rowwise_dot_f32": (c_i, [c_p, c_p, c_l, c_i, c_p, c_p]),
    "tfrs_inbatch_softmax_workspace_bytes": (c_sz, [c_l, c_l, c_i]),
    "tfrs_inbatch_softmax_fwd": (c_i, [c_p, c_p, c_l, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_inbatch_softmax_bwd": (c_i, [c_p, c_p, c_l, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_inbatch_softmax_tc_workspace_bytes": (c_sz, [c_l, c_l, c_i, c_i, c_i]),
    "tfrs_inbatch_softmax_tc_fwd": (c_i, [c_p, c_p, c_l, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_inbatch_softmax_tc_bwd_workspace_bytes": (c_sz, [c_l, c_l, c_i, c_i, c_i]),
    "tfrs_inbatch_softmax_tc_bwd": (c_i, [c_p, c_p, c_l, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_inbatch_softmax_maxsim_workspace_bytes": (c_sz, [c_l, c_i, c_l, c_i]),
    "tfrs_inbatch_softmax_maxsim_fwd": (c_i, [c_p, c_p, c_l, c_i, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_inbatch_softmax_maxsim_bwd": (c_i, [c_p, c_p, c_l, c_i, c_l, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_hardneg_loss_fwd": (c_i, [c_p, c_p, c_l, c_i, c_p, c_f, c_p, c_p, c_p, c_p]),
    "tfrs_hardneg_loss_bwd": (c_i, [c_p, c_p, c_l, c_l, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    "tfrs_sparse_adagrad_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_sparse_adagrad_f32": (c_i, [c_p, c_p, c_l, c_i, c_p, c_i, c_l, c_p, c_f, c_f, c_i, c_p, c_sz, c_p]),
    "tfrs_sparse_clippy_adagrad_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_sparse_clippy_adagrad_f32": (c_i, [c_p, c_p, c_l, c_i, c_p, c_i, c_l, c_p, c_f, c_f, c_f, c_f, c_f, c_i, c_p, c_p, c_sz,
                                             c_p]),
    "tfrs_clippy_adagrad_dense_workspace_bytes": (c_sz, [c_i]),
    "tfrs_clippy_adagrad_dense_f32": (c_i, [c_p, c_p, c_p, c_p, c_i, c_f, c_f, c_f, c_f, c_f, c_i, c_p, c_p, c_sz, c_p]),
    "tfrs_sparse_adam_workspace_bytes": (c_sz, [c_l, c_l]),
    "tfrs_sparse_adam_f32": (c_i, [c_p, c_p, c_p, c_l, c_i, c_p, c_i, c_l, c_p, c_f, c_f, c_f, c_f, c_i, c_p, c_sz, c_p]),
    "tfrs_adam_dense_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_f, c_f, c_f, c_f, c_p]),
    "tfrs_sparse_ftrl_workspace_bytes": (c_sz, [c_l]),
    "tfrs_sparse_ftrl_f32": (c_i, [c_p, c_p, c_p, c_l, c_i, c_p, c_i, c_l, c_p, c_f, c_f, c_f, c_f, c_f, c_p, c_sz, c_p]),
    "tfrs_ftrl_dense_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_f, c_f, c_f, c_f, c_f, c_p]),
    "tfrs_cross_fwd_f32":(c_i, [c_p, c_p, c_p, c_p, c_l, c_i, c_l, c_f, c_p, c_p, c_p]),
    "tfrs_cross_tc_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_cross_tc_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_l, c_i, c_l, c_f, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_cross_bwd_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_cross_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_l, c_i, c_l, c_f, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_cross_tc_bwd_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_cross_tc_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_l, c_i, c_l, c_f, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_gemm_tc_workspace_bytes": (c_sz, [c_l, c_l, c_l]),
    "tfrs_gemm_tc_f32": (c_i, [c_i, c_i, c_l, c_l, c_l, c_p, c_l, c_p, c_l, c_p, c_l, c_p, c_sz, c_p]),
    "tfrs_cross_lowrank_tc_workspace_bytes": (c_sz, [c_l, c_i, c_i]),
    "tfrs_cross_lowrank_tc_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_l, c_i, c_i, c_l, c_f, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_cross_lowrank_tc_bwd_workspace_bytes": (c_sz, [c_l, c_i, c_i]),
    "tfrs_cross_lowrank_tc_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_l, c_i, c_i, c_l, c_f, c_p, c_p, c_p, c_p, c_p,
                                           c_p, c_sz, c_p]),
    "tfrs_dense_uses_tc": (c_i, [c_l, c_i, c_i]),
    "tfrs_dense_fwd_workspace_bytes": (c_sz, [c_l, c_i, c_i]),
    "tfrs_dense_fwd_f32": (c_i, [c_p, c_p, c_p, c_l, c_i, c_i, c_i, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_dense_bwd_workspace_bytes": (c_sz, [c_l, c_i, c_i]),
    "tfrs_dense_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_l, c_i, c_i, c_i, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_ranking_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_ranking_loss_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_l, c_i, c_i, c_p, c_p, c_p, c_f, c_i, c_p, c_sz, c_p]),
    "tfrs_ranking_loss_bwd_f32": (c_i, [c_p, c_p, c_p, c_l, c_i, c_i, c_p, c_p, c_p]),
    "tfrs_ranking_metrics_f32": (c_i, [c_p, c_p, c_p, c_l, c_p, c_f, c_i, c_p, c_sz, c_p]),
    "tfrs_listwise_workspace_bytes": (c_sz, [c_l, c_i]),
    "tfrs_listwise_fwd_f32": (c_i, [c_p, c_p, c_p, c_l, c_i, c_i, c_i, c_f, c_u32, c_u32, c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_p,
                                    c_sz, c_p]),
    "tfrs_listwise_bwd_f32": (c_i, [c_p, c_l, c_i, c_i, c_f, c_p, c_p, c_p]),
    "tfrs_hash_bins": (c_i, [c_p, c_p, c_i, c_l, c_p, c_l, c_p, c_p]),
    "tfrs_unified_lookup_fwd_f32": (c_i, [c_p, c_i, c_p, c_i, c_p]),
    "tfrs_unified_lookup_bwd_f32": (c_i, [c_p, c_i, c_p, c_i, c_p]),
    "tfrs_embedding_bag_fwd_f32": (c_i, [c_p, c_i, c_p]),
    "tfrs_embedding_bag_bwd_f32": (c_i, [c_p, c_i, c_p]),
    "tfrs_sparse_sgd_workspace_bytes": (c_sz, [c_l]),
    "tfrs_sparse_sgd_f32": (c_i, [c_p, c_l, c_i, c_p, c_i, c_l, c_p, c_f, c_p, c_sz, c_p]),
    "tfrs_sgd_dense_f32": (c_i, [c_p, c_p, c_p, c_i, c_f, c_p]),
    "tfrs_tree_ah_assign_workspace_bytes": (c_sz, [c_l, c_i, c_i]),
    "tfrs_tree_ah_assign_f32": (c_i, [c_p, c_l, c_i, c_p, c_i, c_p, c_p, c_sz, c_p]),
    "tfrs_tree_ah_group_workspace_bytes": (c_sz, [c_l]),
    "tfrs_tree_ah_group": (c_i, [c_p, c_l, c_i, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_tree_ah_update_centroids_f32": (c_i, [c_p, c_i, c_p, c_p, c_i, c_p, c_p]),
    "tfrs_tree_ah_init_codebooks_f32": (c_i, [c_p, c_i, c_p, c_p, c_p, c_i, c_p, c_p]),
    "tfrs_tree_ah_encode": (c_i, [c_p, c_i, c_p, c_l, c_p, c_p, c_p, c_i, c_p, c_p]),
    "tfrs_tree_ah_update_codebooks_f32": (c_i, [c_p, c_i, c_l, c_p, c_p, c_p, c_i, c_p, c_p]),
    "tfrs_tree_ah_search_workspace_bytes": (c_sz, [c_l, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_l]),
    "tfrs_tree_ah_search_f32": (c_i, [c_p, c_l, c_i, c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_l, c_p, c_i, c_i, c_i, c_p, c_p,
                                      c_p, c_sz, c_p]),
    "tfrs_lookup_slots": (c_l, [c_l]),
    "tfrs_lookup_table_bytes": (c_sz, [c_l, c_i]),
    "tfrs_lookup_build": (c_i, [c_p, c_p, c_p]),
    "tfrs_lookup": (c_i, [c_p, c_p, c_p, c_i, c_l, c_l, c_l, c_p, c_p, c_p]),
    "tfrs_lookup_invert": (c_i, [c_p, c_i, c_l, c_p, c_l, c_l, c_i, c_l, c_l, c_p, c_p]),
    "tfrs_text_standardize": (c_i, [c_p, c_p, c_l, c_l, c_i, c_p, c_p, c_p, c_p]),
    "tfrs_text_lookup": (c_i, [c_p, c_p, c_p, c_l, c_l, c_l, c_l, c_p, c_p]),
    "tfrs_text_spans": (c_i, [c_p, c_p, c_l, c_p, c_p, c_p]),
    "tfrs_bucketize": (c_i, [c_p, c_i, c_l, c_p, c_l, c_p, c_p]),
    "tfrs_normalize": (c_i, [c_p, c_i, c_l, c_l, c_p, c_p, c_i, c_p, c_p]),
    "tfrs_normalization_adapt_workspace_bytes": (c_sz, [c_l, c_l, c_l]),
    "tfrs_normalization_adapt": (c_i, [c_p, c_i, c_l, c_l, c_l, c_l, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_mean_pool_fwd": (c_i, [c_p, c_l, c_l, c_l, c_l, c_l, c_l, c_p, c_i, c_p, c_p]),
    "tfrs_mean_pool_bwd": (c_i, [c_p, c_l, c_l, c_l, c_p, c_i, c_p, c_p]),
    "tfrs_hashing": (c_i, [c_p, c_p, c_i, c_l, c_p, c_l, c_i, c_l, c_p, c_l, c_p, c_p]),
    "tfrs_gru_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_l, c_l, c_i, c_p, c_p, c_p, c_p, c_p]),
    "tfrs_gru_bwd_workspace_bytes": (c_sz, [c_l, c_l, c_i]),
    "tfrs_gru_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_l, c_l, c_i, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_lstm_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_l, c_l, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p]),
    "tfrs_lstm_bwd_workspace_bytes": (c_sz, [c_l, c_l, c_i]),
    "tfrs_lstm_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_l, c_l, c_i, c_p, c_p, c_p, c_p, c_p,
                                c_sz, c_p]),
    "tfrs_mha_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_l, c_l, c_l, c_i, c_i, c_i, c_p, c_p, c_p, c_p]),
    "tfrs_mha_bwd_workspace_bytes": (c_sz, [c_l, c_l, c_i]),
    "tfrs_mha_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_l, c_l, c_l, c_i, c_i, c_i, c_p, c_p, c_p, c_p, c_sz,
                               c_p]),
    "tfrs_dense_attention_fwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_l, c_l, c_l, c_i, c_i, c_p, c_p, c_p, c_p]),
    "tfrs_dense_attention_bwd_workspace_bytes": (c_sz, [c_i, c_l, c_l, c_i]),
    "tfrs_dense_attention_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_l, c_l, c_l, c_i, c_i, c_p, c_p, c_p, c_p,
                                           c_p, c_p, c_sz, c_p]),
    "tfrs_layer_norm_fwd_f32": (c_i, [c_p, c_p, c_p, c_l, c_l, c_f, c_p, c_p, c_p, c_p]),
    "tfrs_layer_norm_bwd_workspace_bytes": (c_sz, [c_l, c_l]),
    "tfrs_layer_norm_bwd_f32": (c_i, [c_p, c_p, c_p, c_p, c_p, c_l, c_l, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_dropout_f32": (c_i, [c_p, c_i, c_p, c_p, c_d, c_u64, c_u64, c_p, c_p]),
    "tfrs_batch_norm_fwd_workspace_bytes": (c_sz, [c_l, c_l]),
    "tfrs_batch_norm_fwd_f32": (c_i, [c_p, c_p, c_i, c_p, c_p, c_l, c_l, c_i, c_d, c_f, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "tfrs_batch_norm_bwd_workspace_bytes": (c_sz, [c_l, c_l]),
    "tfrs_batch_norm_bwd_f32": (c_i, [c_p, c_p, c_i, c_p, c_p, c_p, c_l, c_l, c_i, c_p, c_p, c_p, c_sz, c_p]),
}

EXPORTS = tuple(_SIGNATURES)


def lib() -> ctypes.CDLL:
  """Loads libtfrs_b200.so; raises (never falls back) when it is missing."""
  global _lib
  if _lib is None:
    if not os.path.exists(LIB_PATH):
      raise RuntimeError(
          f"libtfrs_b200.so not found at {LIB_PATH}. Build it with `python -m recommenders_b200.build` "
          "(nvcc, sm_90a). There is no CPU fallback.")
    l = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
      fn = getattr(l, name)  # AttributeError if the symbol is missing: fail loudly
      fn.restype = res
      fn.argtypes = args
    _lib = l
  return _lib


def last_error() -> str:
  return lib().tfrs_last_error().decode("utf-8", "replace")


def check(rc: int, what: str = "") -> None:
  if rc == 0:
    return
  msg = f"{what}: {last_error()} (code {rc})" if what else f"{last_error()} (code {rc})"
  if rc == -1:
    raise ValueError(msg)
  if rc == -2:
    raise NotImplementedError(msg)
  if rc == -5:
    raise RuntimeError("NCCL: " + msg)
  raise RuntimeError(msg)


def require_cuda(t: torch.Tensor, name: str) -> torch.Tensor:
  if not isinstance(t, torch.Tensor):
    raise TypeError(f"{name} must be a torch.Tensor, got {type(t)}")
  if not t.is_cuda:
    raise RuntimeError(f"{name} must live on a CUDA device (got {t.device}); recommenders_b200 has no CPU path.")
  return t


def f32c(t: torch.Tensor, name: str) -> torch.Tensor:
  require_cuda(t, name)
  if t.dtype != torch.float32:
    t = t.to(torch.float32)
  return t.contiguous()


def ptr(t: Optional[torch.Tensor]):
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream() -> ctypes.c_void_p:
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


_ws_cache = {}          # (device, stream, slot) -> uint8 tensor; insertion order = recency (re-inserted on every use)
_WS_CACHE_MAX = 64      # entries; the least recently used buffers are dropped beyond this (streams come and go)


def workspace(nbytes: int, device: torch.device, slot: str = "default") -> torch.Tensor:
  """A per-(device, stream, slot) scratch buffer that only grows (caller-provided scratch of the C ABI).  The cache is
  bounded: least-recently-used entries are dropped (the caching allocator keeps a dropped buffer alive until the work
  already enqueued on its stream has finished)."""
  key = (device.index if device.index is not None else torch.cuda.current_device(),
         torch.cuda.current_stream().cuda_stream, slot)
  buf = _ws_cache.pop(key, None)
  if buf is None or buf.numel() < nbytes:
    buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
  _ws_cache[key] = buf
  while len(_ws_cache) > _WS_CACHE_MAX:
    _ws_cache.pop(next(iter(_ws_cache)))
  return buf


def release_workspaces() -> None:
  """Drops every cached scratch buffer (e.g. after an evaluation pass whose shapes will not come back)."""
  _ws_cache.clear()


def ids_dtype_code(t: torch.Tensor) -> int:
  if t.dtype == torch.int32:
    return I32
  if t.dtype == torch.int64:
    return I64
  raise TypeError(f"ids must be int32 or int64, got {t.dtype}")
