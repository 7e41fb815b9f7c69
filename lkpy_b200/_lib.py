"""
ctypes binding of the C ABI declared in ``include/lkpy_b200.h``.

Loading fails loudly: there is no CPU or PyTorch fallback behind these entry
points.  ``lib()`` needs the built ``.so`` (``python -m lkpy_b200._build``);
``require_device()`` additionally needs a CUDA device.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "csrc" / "liblkpy_b200.so"

LK_OK = 0
LK_DTYPE_F32, LK_DTYPE_BF16 = 0, 1
LK_ALS_IMPLICIT, LK_ALS_EXPLICIT = 0, 1
LK_MAX_REPLICAS = 8
LK_COOC_COUNT, LK_ASSOC_PROBABILITY, LK_ASSOC_LIFT = 0, 1, 2
LK_FLEXMF_LOGISTIC, LK_FLEXMF_PAIRWISE, LK_FLEXMF_MSE = 0, 1, 2
LK_FLEXMF_REG_NONE, LK_FLEXMF_REG_L2, LK_FLEXMF_REG_ADAMW = 0, 1, 2
LK_STOCH_NONE, LK_STOCH_SOFTMAX, LK_STOCH_LINEAR = 0, 1, 2
LK_STOCH_JUMP_WORDS = 4 * (33 + 64)
LK_FAIR_LISTS, LK_FAIR_SCORES = 0, 1
(LK_METRIC_HIT, LK_METRIC_PRECISION, LK_METRIC_RECALL, LK_METRIC_RECIP_RANK, LK_METRIC_DCG, LK_METRIC_NDCG,
 LK_METRIC_RBP, LK_METRIC_AP, LK_METRIC_MEAN_POP_RANK) = range(9)  # fmt: skip
LK_RBP_NORM_SERIES, LK_RBP_NORM_PREFIX, LK_RBP_NORM_LIST = 0, 1, 2
LK_RANK_METRICS_MAX = 32

i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
u64p = C.POINTER(C.c_uint64)
vp = C.c_void_p


class EngineError(RuntimeError):
    """An error reported by the CUDA library."""


class LkAlsArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int32),
        ("k", C.c_int32),
        ("n_rows", C.c_int64),
        ("n_other", C.c_int64),
        ("d_indptr", vp),
        ("d_cols", vp),
        ("d_vals", vp),
        ("d_this", vp),
        ("d_other", vp),
        ("other_dtype", C.c_int32),
        ("n_replicas", C.c_int32),
        ("d_replicas", vp * LK_MAX_REPLICAS),
        ("replica_row0", C.c_int64),
        ("d_otor", vp),
        ("reg", C.c_float),
        ("d_chunks", vp),
        ("n_chunks", C.c_int64),
        ("d_partials", vp),
        ("d_split_counters", vp),
        ("n_split_rows", C.c_int64),
        ("d_work_counter", vp),
        ("d_sqdelta", vp),
        ("d_status", vp),
        ("vals_uniform", C.c_int32),
        ("uniform_val", C.c_float),
        ("d_cancel", vp),
    ]


class LkKnnGeom(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("warps", C.c_int32),
        ("tile_cols", C.c_int32),
        ("n_halves", C.c_int32),
        ("n_subtiles", C.c_int32),
        ("smem_bytes", C.c_int32),
        ("ctas_per_sm", C.c_int32),
    ]


class LkKnnBuildArgs(C.Structure):
    _fields_ = [
        ("geom", LkKnnGeom),
        ("d_ui_indptr", vp),
        ("d_ui_cols", vp),
        ("d_ui_vals", vp),
        ("d_iu_indptr", vp),
        ("d_iu_cols", vp),
        ("d_iu_vals", vp),
        ("d_tile_ptr", vp),
        ("d_units", vp),
        ("d_unit_ptr", vp),
        ("max_units_per_item", C.c_int32),
        ("d_sched", vp),
        ("n_work", C.c_int64),
        ("min_sim", C.c_float),
        ("save_nbrs", C.c_int32),
        ("d_part_cols", vp),
        ("d_part_vals", vp),
        ("d_part_cnt", vp),
        ("d_pool_cols", vp),
        ("d_pool_vals", vp),
        ("pool_capacity", C.c_int64),
        ("d_pool_off", vp),
        ("d_pool_cursor", vp),
        ("d_tie_scratch", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_cancel", vp),
    ]


class LkKnnScoreArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int32),
        ("d_sim_indptr", vp),
        ("d_sim_cols", vp),
        ("d_sim_vals", vp),
        ("n_queries", C.c_int32),
        ("d_ref_indptr", vp),
        ("d_ref_items", vp),
        ("d_ref_vals", vp),
        ("d_tgt_indptr", vp),
        ("d_tgt_items", vp),
        ("max_nbrs", C.c_int32),
        ("min_nbrs", C.c_int32),
        ("d_slotmap", vp),
        ("slotmap_warps", C.c_int64),
        ("d_list_off", vp),
        ("d_list_cur", vp),
        ("d_list_cnt", vp),
        ("d_scores", vp),
        ("d_counts", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_pool", vp),
        ("pool_entries", C.c_int64),
        ("d_pool_cursor", vp),
        ("user_mode", C.c_int32),
        ("n_matrix_rows", C.c_int32),
    ]


class LkKnnRankArgs(C.Structure):
    _fields_ = [
        ("n", C.c_int32),
        ("d_item_offset", vp),
        ("d_query_offset", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_spill", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_nbrs", vp),
        ("d_out_cnt", vp),
    ]


class LkUknnSearchArgs(C.Structure):
    _fields_ = [
        ("geom", LkKnnGeom),
        ("d_vt_indptr", vp),
        ("d_vt_users", vp),
        ("d_vt_vals", vp),
        ("d_tile_ptr", vp),
        ("n_queries", C.c_int32),
        ("d_q_begin", vp),
        ("d_q_end", vp),
        ("d_q_items", vp),
        ("d_q_vals", vp),
        ("d_q_self", vp),
        ("min_sim", C.c_double),
        ("d_sched", vp),
        ("n_work", C.c_int64),
        ("d_pool_rows", vp),
        ("d_pool_sims", vp),
        ("pool_capacity", C.c_int64),
        ("d_pool_off", vp),
        ("d_part_cnt", vp),
        ("d_pool_cursor", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
    ]


class LkAlsRecArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int64),
        ("k", C.c_int32),
        ("n_queries", C.c_int32),
        ("d_items", vp),
        ("d_queries", vp),
        ("d_item_offset", vp),
        ("d_query_offset", vp),
        ("n", C.c_int32),
        ("d_scores", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_workspace", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_cnt", vp),
    ]


class LkCoocArgs(C.Structure):
    _fields_ = [
        ("geom", LkKnnGeom),
        ("d_gi_indptr", vp),
        ("d_gi_items", vp),
        ("d_ig_indptr", vp),
        ("d_ig_groups", vp),
        ("d_tile_ptr", vp),
        ("full_rows", C.c_int32),
        ("method", C.c_int32),
        ("d_item_count", vp),
        ("damping", C.c_double),
        ("max_row_cost", C.c_int64),
        ("d_sched", vp),
        ("n_work", C.c_int64),
        ("d_pool_cols", vp),
        ("d_pool_vals", vp),
        ("pool_capacity", C.c_int64),
        ("d_pool_off", vp),
        ("d_part_cnt", vp),
        ("d_pool_cursor", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_cancel", vp),
    ]


class LkAssocScoreArgs(C.Structure):
    _fields_ = [
        ("geom", LkKnnGeom),
        ("d_indptr", vp),
        ("d_cols", vp),
        ("d_vals", vp),
        ("d_tile_ptr", vp),
        ("n_queries", C.c_int32),
        ("agg", C.c_int32),
        ("d_ref_indptr", vp),
        ("d_ref_items", vp),
        ("n", C.c_int32),
        ("d_scores", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_cnt", vp),
    ]


class LkEaseScoreArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int32),
        ("d_w", vp),
        ("n_queries", C.c_int32),
        ("d_hist_indptr", vp),
        ("d_hist_items", vp),
        ("n", C.c_int32),
        ("d_scores", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_cnt", vp),
    ]


class LkSlimArgs(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("d_ui_indptr", vp),
        ("d_ui_cols", vp),
        ("d_iu_indptr", vp),
        ("d_iu_cols", vp),
        ("l1_reg", C.c_float),
        ("l2_reg", C.c_float),
        ("max_iters", C.c_int32),
        ("max_nbrs", C.c_int32),
        ("d_sched", vp),
        ("n_work", C.c_int64),
        ("d_workspace", vp),
        ("workspace_bytes", C.c_int64),
        ("d_pool_cols", vp),
        ("d_pool_vals", vp),
        ("pool_capacity", C.c_int64),
        ("d_pool_off", vp),
        ("d_part_cnt", vp),
        ("d_pool_cursor", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_cancel", vp),
    ]


class LkFlexmfSampleArgs(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("d_ui_indptr", vp),
        ("d_ui_cols", vp),
        ("d_coo_items", vp),
        ("nnz", C.c_int64),
        ("d_rows", vp),
        ("n_samples", C.c_int64),
        ("batch_size", C.c_int32),
        ("n", C.c_int32),
        ("max_attempts", C.c_int32),
        ("popular", C.c_int32),
        ("seed", C.c_uint64),
        ("step0", C.c_int64),
        ("d_out", vp),
    ]


class LkFlexmfGroups(C.Structure):
    _fields_ = [
        ("d_occ", vp),
        ("d_unit_start", vp),
        ("d_unit_uniq", vp),
        ("d_uniq_row", vp),
        ("d_uniq_unit", vp),
        ("unit0", C.c_int64),
        ("uniq0", C.c_int64),
        ("n_uniq", C.c_int32),
        ("d_mark", vp),
    ]


class LkFlexmfStepArgs(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("k", C.c_int32),
        ("batch", C.c_int32),
        ("n_neg", C.c_int32),
        ("loss", C.c_int32),
        ("reg_method", C.c_int32),
        ("positive_weight", C.c_float),
        ("regularization", C.c_float),
        ("decay", C.c_float),
        ("one_minus_beta1", C.c_float),
        ("beta2", C.c_float),
        ("one_minus_beta2", C.c_float),
        ("eps", C.c_float),
        ("step_size", C.c_float),
        ("bias2_sqrt", C.c_float),
        ("step", C.c_int64),
        ("d_u_emb", vp), ("d_u_emb_m", vp), ("d_u_emb_v", vp),
        ("d_i_emb", vp), ("d_i_emb_m", vp), ("d_i_emb_v", vp),
        ("d_u_bias", vp), ("d_u_bias_m", vp), ("d_u_bias_v", vp),
        ("d_i_bias", vp), ("d_i_bias_m", vp), ("d_i_bias_v", vp),
        ("d_users", vp),
        ("d_pos", vp),
        ("d_neg", vp),
        ("u_groups", LkFlexmfGroups),
        ("i_groups", LkFlexmfGroups),
        ("n_u_units", C.c_int32),
        ("n_i_units", C.c_int32),
        ("d_workspace", vp),
        ("workspace_bytes", C.c_int64),
        ("d_loss", vp),
        ("d_ratings", vp),
    ]  # fmt: skip


class LkSpmmArgs(C.Structure):
    _fields_ = [
        ("n_rows", C.c_int32),
        ("n_src", C.c_int32),
        ("width", C.c_int32),
        ("nnz", C.c_int64),
        ("d_indptr", vp),
        ("d_indices", vp),
        ("d_values", vp),
        ("d_order", vp),
        ("d_dense", vp),
        ("d_out", vp),
    ]


class LkNmfCdSweepArgs(C.Structure):
    _fields_ = [
        ("n", C.c_int32),
        ("k", C.c_int32),
        ("d_w", vp),
        ("d_hht", vp),
        ("d_xht", vp),
        ("d_pg", vp),
    ]


class LkF32SeqSumArgs(C.Structure):
    _fields_ = [
        ("n", C.c_int64),
        ("d_x", vp),
        ("d_out", vp),
    ]


class LkBiasLearnArgs(C.Structure):
    _fields_ = [
        ("nnz", C.c_int64),
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("d_ratings", vp),
        ("d_items", vp),
        ("d_user_indptr", vp),
        ("d_item_indptr", vp),
        ("d_item_ratings", vp),
        ("d_user_order", vp),
        ("d_item_order", vp),
        ("centered_f64", C.c_int32),
        ("damping_user", C.c_double),
        ("damping_item", C.c_double),
        ("d_workspace", vp),
        ("d_mean", vp),
        ("d_item_bias", vp),
        ("d_user_bias", vp),
    ]


class LkOffsetScoreArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int32),
        ("n_queries", C.c_int32),
        ("d_base", vp),
        ("d_offset", vp),
        ("n", C.c_int32),
        ("d_scores", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_cnt", vp),
    ]


class LkStochasticArgs(C.Structure):
    _fields_ = [
        ("n_queries", C.c_int32),
        ("n_items", C.c_int32),
        ("d_scores", vp),
        ("row_stride", C.c_int64),
        ("item_stride", C.c_int64),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("transform", C.c_int32),
        ("scale", C.c_float),
        ("shared_stream", C.c_int32),
        ("n", C.c_int32),
        ("d_state", vp),
        ("d_jump", vp),
        ("d_position", vp),
        ("d_workspace", vp),
        ("workspace_bytes", C.c_int64),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_key", vp),
        ("d_out_cnt", vp),
        ("d_keys", vp),
    ]


class LkFairArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int32),
        ("n_queries", C.c_int32),
        ("n", C.c_int32),
        ("n_candidates", C.c_int32),
        ("d_m", vp),
        ("d_list_indptr", vp),
        ("d_list_protected", vp),
        ("d_list_len", vp),
        ("n_items", C.c_int32),
        ("d_scores", vp),
        ("row_stride", C.c_int64),
        ("item_stride", C.c_int64),
        ("d_item_protected", vp),
        ("d_excl_indptr", vp),
        ("d_excl_items", vp),
        ("d_out_idx", vp),
        ("d_out_val", vp),
        ("d_out_cnt", vp),
    ]


class LkMetricSpec(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("n", C.c_int32),
        ("weight_offset", C.c_int64),
        ("norm_offset", C.c_int64),
        ("norm_mode", C.c_int32),
        ("reserved", C.c_int32),
        ("series_sum", C.c_double),
    ]


class LkRankMetricsArgs(C.Structure):
    _fields_ = [
        ("n_lists", C.c_int64),
        ("d_rec_indptr", vp),
        ("d_rec_items", vp),
        ("d_test_indptr", vp),
        ("d_test_items", vp),
        ("d_nrel", vp),
        ("d_weights", vp),
        ("d_norms", vp),
        ("d_out", vp),
        ("n_metrics", C.c_int32),
        ("reserved", C.c_int32),
        ("metrics", LkMetricSpec * LK_RANK_METRICS_MAX),
    ]


class LkItemExposureArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int64),
        ("n_entries", C.c_int64),
        ("d_sorted_items", vp),
        ("d_order", vp),
        ("d_entry_list", vp),
        ("d_entry_rank", vp),
        ("d_weights", vp),
        ("d_totals", vp),
    ]


#: every symbol ``include/lkpy_b200.h`` declares: name -> (restype, argtypes)
SYMBOLS: dict[str, tuple] = {
    "lk_version": (C.c_int, []),
    "lk_last_error": (C.c_char_p, []),
    "lk_device_info": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "lk_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "lk_get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    "lk_als_max_features": (C.c_int, []),
    "lk_als_plan_size": (C.c_int, [vp, C.c_int64, C.c_int32, i64p, i64p, i64p]),
    "lk_als_plan_fill": (C.c_int, [vp, C.c_int64, C.c_int32, vp]),
    "lk_als_slot_floats": (C.c_int64, [C.c_int32]),
    "lk_als_half_epoch": (C.c_int, [C.POINTER(LkAlsArgs), vp]),
    "lk_als_otor_scratch_floats": (C.c_int64, [C.c_int32]),
    "lk_als_otor": (C.c_int, [vp, C.c_int64, C.c_int32, C.c_float, vp, vp, vp, vp]),
    "lk_knn_geometry": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(LkKnnGeom)]),
    "lk_knn_tile_pointers": (C.c_int, [C.POINTER(LkKnnGeom), vp, vp, vp, vp]),
    "lk_knn_row_cost": (C.c_int, [C.POINTER(LkKnnGeom), vp, vp, vp, vp, vp]),
    "lk_knn_tie_scratch_ints": (C.c_int64, [C.POINTER(LkKnnGeom)]),
    "lk_knn_build": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp]),
    "lk_knn_merge_topk": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp, vp, vp, vp]),
    "lk_knn_pool_to_csr": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp, vp, vp, vp]),
    "lk_uknn_geometry": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(LkKnnGeom)]),
    "lk_uknn_query_cost": (C.c_int, [C.POINTER(LkUknnSearchArgs), vp, vp]),
    "lk_uknn_search": (C.c_int, [C.POINTER(LkUknnSearchArgs), vp]),
    "lk_uknn_pool_to_csr": (C.c_int, [C.POINTER(LkUknnSearchArgs), vp, vp, vp, vp]),
    "lk_knn_prep_columns": (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    "lk_knn_score_warps": (C.c_int64, []),
    "lk_knn_score_dense_ctas": (C.c_int64, []),
    "lk_knn_score_batch": (C.c_int, [C.POINTER(LkKnnScoreArgs), vp]),
    "lk_knn_recommend_batch": (C.c_int, [C.POINTER(LkKnnScoreArgs), C.POINTER(LkKnnRankArgs), vp]),
    "lk_topn_max": (C.c_int, []),
    "lk_topn_columns": (C.c_int, [vp, C.c_int64, C.c_int64, C.c_int64, C.c_int32, vp, vp, vp, vp]),
    "lk_als_recommend_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "lk_als_recommend_batch": (C.c_int, [C.POINTER(LkAlsRecArgs), vp]),
    "lk_cooc_geometry": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(LkKnnGeom)]),
    "lk_cooc_row_cost": (C.c_int, [C.POINTER(LkCoocArgs), vp, vp]),
    "lk_cooc_count": (C.c_int, [C.POINTER(LkCoocArgs), vp]),
    "lk_cooc_pool_to_csr": (C.c_int, [C.POINTER(LkCoocArgs), vp, vp, vp, vp]),
    "lk_cooc_diagonal": (C.c_int, [C.POINTER(LkCoocArgs), vp, vp]),
    "lk_cooc_dense": (C.c_int, [C.c_int32, vp, vp, vp, vp, vp, vp]),
    "lk_assoc_tile_pointers": (C.c_int, [C.POINTER(LkKnnGeom), vp, vp, vp, vp]),
    "lk_assoc_score_batch": (C.c_int, [C.POINTER(LkAssocScoreArgs), vp]),
    "lk_ease_score_batch": (C.c_int, [C.POINTER(LkEaseScoreArgs), vp]),
    "lk_slim_workspace_bytes": (C.c_int, [C.c_int32, C.c_int32, C.c_int64, i64p]),
    "lk_slim_train": (C.c_int, [C.POINTER(LkSlimArgs), vp]),
    "lk_slim_pool_to_csr": (C.c_int, [C.POINTER(LkSlimArgs), vp, vp, vp, vp]),
    "lk_flexmf_sample_negatives": (C.c_int, [C.POINTER(LkFlexmfSampleArgs), vp]),
    "lk_flexmf_workspace_bytes": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, i64p]),
    "lk_flexmf_step": (C.c_int, [C.POINTER(LkFlexmfStepArgs), vp]),
    "lk_spmm": (C.c_int, [C.POINTER(LkSpmmArgs), vp]),
    "lk_nmf_cd_sweep": (C.c_int, [C.POINTER(LkNmfCdSweepArgs), vp]),
    "lk_f32_seq_sum": (C.c_int, [C.POINTER(LkF32SeqSumArgs), C.c_int32, vp]),
    "lk_bias_learn_workspace_bytes": (C.c_int64, []),
    "lk_bias_learn": (C.c_int, [C.POINTER(LkBiasLearnArgs), vp]),
    "lk_offset_score_batch": (C.c_int, [C.POINTER(LkOffsetScoreArgs), vp]),
    "lk_stochastic_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32]),
    "lk_stochastic_topn": (C.c_int, [C.POINTER(LkStochasticArgs), vp]),
    "lk_fair_rerank": (C.c_int, [C.POINTER(LkFairArgs), vp]),
    "lk_rank_metrics": (C.c_int, [C.POINTER(LkRankMetricsArgs), vp]),
    "lk_item_exposure": (C.c_int, [C.POINTER(LkItemExposureArgs), vp]),
}

_lib = None


def lib():
    """Load the CUDA library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise EngineError(
                f"{LIB_PATH} is missing: build it with `python -m lkpy_b200._build` "
                "(there is no CPU fallback for the lkpy_b200 engines)"
            )
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def set_option(name: str, value: int) -> None:
    """Switch a diagnostic kernel variant (``lk_set_option``; the LK_* environment is read once at load)."""
    check(lib().lk_set_option(name.encode(), int(value)), "lk_set_option")


def get_option(name: str) -> int:
    v = C.c_int()
    check(lib().lk_get_option(name.encode(), C.byref(v)), "lk_get_option")
    return int(v.value)


def check(rc: int, what: str = "") -> None:
    if rc != LK_OK:
        msg = lib().lk_last_error().decode("utf-8", "replace")
        raise EngineError(f"{what or 'lkpy_b200'} failed (code {rc}): {msg}")


def require_device():
    """The torch CUDA device the engines run on; raises without one."""
    import torch

    if not torch.cuda.is_available():
        raise EngineError(
            "lkpy_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback"
        )
    return torch.device("cuda", torch.cuda.current_device())


def ptr(t) -> int | None:
    """Device (or host) address of a torch tensor / NumPy array, None for None."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def stream_ptr() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
