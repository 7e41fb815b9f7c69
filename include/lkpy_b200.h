/*
 * lkpy_b200.h — C ABI of the H100-native ALS / item-kNN engine.
 *
 * This is the drop-in boundary for the reference's native accelerator
 * `lenskit._accel` (PyO3 cdylib, src/accel/lib.rs:25-49) restricted to the two
 * hot paths:
 *
 *   reference entry point                         (file:line)                      replaced by
 *   -------------------------------------------------------------------------------------------------
 *   _accel.als.train_implicit_matrix              src/accel/als/implicit.rs:35-53   lk_als_half_epoch (mode 0)
 *   _accel.als.train_explicit_matrix              src/accel/als/explicit.rs:35-52   lk_als_half_epoch (mode 1)
 *   _implicit_otor (NumPy, host)                  src/lenskit/als/_implicit.py:177  lk_als_otor
 *   POSV::solve (LAPACK sposv)                    src/accel/als/solve.rs:65-106     in-kernel Cholesky
 *   _accel.knn.compute_similarities               src/accel/knn/item_train.rs:32-93 lk_knn_geometry + lk_knn_build
 *   _accel.knn.score_explicit / score_implicit    src/accel/knn/item_score.rs:22-111 lk_knn_score_batch
 *   kNN scorer + TopNRanker (topn_pipeline)       src/lenskit/basic/topn.py:32-69   lk_knn_recommend_batch
 *   UserKNNScorer neighbours (SciPy, host)        src/lenskit/knn/user.py:189-214   lk_uknn_search
 *   _accel.data.argtopn (SURVEY.md 8f, "next")    src/accel/data/sorting.rs:131-170 lk_topn_columns
 *   ALS scorer + TopNRanker (score_matrix/recommend_batch) src/lenskit/als/_common.py:133-175 lk_als_recommend_batch
 *   _accel.data.count_cooc / dense_cooc           src/accel/data/cooc.rs:49-214     lk_cooc_count (+ _diagonal, _dense)
 *   AssociationScorer.train / __call__            src/lenskit/knn/association.py    lk_cooc_count (LK_ASSOC_*), lk_assoc_score_batch
 *   EASEScorer.__call__ (q_vec @ weights)         src/lenskit/knn/ease.py           lk_ease_score_batch
 *   _accel.slim.train_slim                        src/accel/slim/mod.rs:57-93       lk_slim_train (+ lk_slim_pool_to_csr)
 *   SLIMScorer.__call__ (x @ weights)             src/lenskit/knn/slim.py           lk_assoc_score_batch (agg 2)
 *   sample_negatives (host, per minibatch)        src/accel/data/sampling.rs:38-58  lk_flexmf_sample_negatives
 *   FlexMFImplicitTrainer.train_batch (autograd)  src/lenskit/flexmf/_implicit.py:253-274 lk_flexmf_step
 *   FlexMFExplicitTrainer.train_batch (autograd)  src/lenskit/flexmf/_explicit.py:108-125 lk_flexmf_step (LK_FLEXMF_MSE)
 *   FlexMFScorerBase.__call__ + TopNRanker        src/lenskit/flexmf/_base.py:117-157 lk_als_recommend_batch (biases as offsets)
 *   TruncatedSVD sparse products (SciPy, host)    src/lenskit/sklearn/svd.py         lk_spmm
 *   BiasedSVDScorer.__call__ + TopNRanker         src/lenskit/sklearn/svd.py         lk_als_recommend_batch (biases as offsets)
 *   NMFScorer.train (scikit-learn _update_cdnmf_fast) src/lenskit/sklearn/nmf.py     lk_nmf_cd_sweep + lk_f32_seq_sum (+ lk_spmm)
 *   NMFScorer.__call__ + TopNRanker               src/lenskit/sklearn/nmf.py         lk_als_recommend_batch
 *   BiasModel.learn (NumPy, host)                 src/lenskit/basic/bias.py:84-150   lk_bias_learn
 *   BiasScorer / PopScorer __call__ + TopNRanker  src/lenskit/basic/bias.py, popularity.py lk_offset_score_batch
 *   StochasticTopNRanker.__call__ (_compute_keys + ItemList.top_n)
 *                                                 src/lenskit/stochastic/_ranker.py:89-156,
 *                                                 src/lenskit/data/_items.py:942-998 lk_stochastic_topn
 *   FAIRReranker.__call__ (and TopNRanker + FAIRReranker)
 *                                                 src/lenskit/reranking/fair.py      lk_fair_rerank
 *   MeasurementCollector over the ranking metrics (measure_list per list and metric)
 *                                                 src/lenskit/metrics/ranking/*.py   lk_rank_metrics, lk_item_exposure
 *
 * Conventions
 *   - plain C: pointers and sizes only; no C++/torch types cross this boundary;
 *   - pointers named d_* are DEVICE pointers (owned by the caller, e.g. torch
 *     tensors), h_* are HOST pointers; the library never allocates or frees
 *     device memory — every workspace is sized by a *_plan_* / *_workspace_*
 *     call and passed in;
 *   - `stream` is a cudaStream_t passed as void*; all device work is enqueued
 *     on it and nothing synchronises unless stated;
 *   - every function returns LK_OK (0) or a negative LK_ERR_* code and never
 *     throws; lk_last_error() gives a thread-local message.  Numerical failure
 *     (a non positive-definite ALS system, the reference's
 *     RuntimeError("ALS solve error…"), implicit.rs:79) is reported through a
 *     device status word so that no sync is forced.
 *   - CSR matrices are three arrays exactly like the reference's Arrow
 *     List<Struct{index:i32,value:f32}> storage (src/accel/sparse/csr.rs:160-209):
 *     offsets (int32), column indices (int32, ascending within a row), values (f32).
 */
#ifndef LKPY_B200_H
#define LKPY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LK_OK 0
#define LK_ERR_INVALID (-1)     /* bad argument */
#define LK_ERR_CUDA (-2)        /* CUDA runtime error (see lk_last_error) */
#define LK_ERR_UNSUPPORTED (-3) /* shape outside what the kernels cover */
#define LK_ERR_NO_DEVICE (-4)   /* no CUDA device / wrong architecture */

#define LK_DTYPE_F32 0
#define LK_DTYPE_BF16 1

#define LK_ALS_IMPLICIT 0
#define LK_ALS_EXPLICIT 1

#define LK_MAX_REPLICAS 8

#if defined(__GNUC__)
#define LK_API __attribute__((visibility("default")))
#else
#define LK_API
#endif

LK_API int lk_version(void);
LK_API const char *lk_last_error(void);
/* Number of SMs and compute capability (major*10+minor) of the current device. */
LK_API int lk_device_info(int *sm_count, int *cc);
/* Diagnostic switches (kernel variants kept for comparison; none changes results beyond rounding).
 * Each is also an environment variable of the same name, read once when the library first needs
 * it — never per launch; after that only lk_set_option changes it.  Names: LK_ALS_TC,
 * LK_ALS_TF32, LK_KNN_WARPS, LK_KNN_CTAS, LK_KNN_SCORE_CTAS (meaning: lkpy_b200/csrc/common.cuh, struct Options). */
LK_API int lk_set_option(const char *name, int value);
LK_API int lk_get_option(const char *name, int *value);

/* ------------------------------------------------------------------------- */
/* ALS                                                                        */
/* ------------------------------------------------------------------------- */

/* Largest embedding size the kernels cover (padded internally to 32/64/128). */
LK_API int lk_als_max_features(void);

/*
 * Row scheduling plan (host side, once per matrix).  Rows are cut into chunks
 * of at most `chunk_nnz` nonzeros so that power-law rows neither serialise on
 * one warp nor unbalance the grid; chunks are ordered longest-row-first.
 * `chunk_nnz` must be a positive multiple of 32 (else LK_ERR_INVALID); a row
 * longer than it is cut into ceil(n / chunk_nnz) parts of 1 .. chunk_nnz
 * nonzeros each (equal lengths rounded up to 32, the last part shorter).  Each
 * chunk record is 8 int32:
 *   {row, nnz_begin, nnz_len, n_parts, first_slot, part_index, split_index, 0}
 * n_parts == 1 for a whole row.  Rows split into several chunks accumulate
 * partial Gram matrices in `d_partials` and the last part to finish reduces
 * them in slot order (deterministic) and solves.
 *
 * lk_als_plan_size: returns the number of chunks, split rows and partial slots.
 * lk_als_plan_fill: fills h_chunks [n_chunks*8].
 */
LK_API int lk_als_plan_size(const int32_t *h_indptr, int64_t n_rows, int32_t chunk_nnz,
                     int64_t *n_chunks, int64_t *n_split_rows, int64_t *n_slots);
LK_API int lk_als_plan_fill(const int32_t *h_indptr, int64_t n_rows, int32_t chunk_nnz,
                     int32_t *h_chunks);
/* floats needed per partial slot for embedding size k */
LK_API int64_t lk_als_slot_floats(int32_t k);

typedef struct lk_als_args {
    int32_t mode;            /* LK_ALS_IMPLICIT | LK_ALS_EXPLICIT */
    int32_t k;               /* embedding size (row length of this/other) */
    int64_t n_rows;          /* rows of the matrix / of `this` */
    int64_t n_other;         /* rows of `other` */
    const int32_t *d_indptr; /* [n_rows+1] */
    const int32_t *d_cols;   /* [nnz] */
    const float *d_vals;     /* [nnz] (implicit: confidence incl. weight; explicit: bias-removed rating) */
    float *d_this;           /* [n_rows,k] f32, updated in place (implicit.rs:57-58) */
    const void *d_other;     /* [n_other,k] f32 or bf16 (other_dtype), read only */
    int32_t other_dtype;     /* LK_DTYPE_* */
    int32_t n_replicas;      /* extra copies of `this` to write (peer GPUs); 0 on one GPU */
    float *d_replicas[LK_MAX_REPLICAS]; /* each [*, k] f32; row r goes to d_replicas[i] + (replica_row0 + r)*k */
    int64_t replica_row0;    /* row offset of this shard inside the replicas */
    const float *d_otor;     /* [k,k] f32: O^T O + reg I (implicit) or NULL */
    float reg;               /* explicit: A += reg * nnz(row) * I (explicit.rs:106-108) */
    const int32_t *d_chunks; /* plan, [n_chunks*8] */
    int64_t n_chunks;
    float *d_partials;       /* [n_slots * lk_als_slot_floats(k)] or NULL if no split rows */
    int32_t *d_split_counters; /* [n_split_rows] zeroed by the call */
    int64_t n_split_rows;
    int32_t *d_work_counter; /* [1] zeroed by the call */
    double *d_sqdelta;       /* [1] += sum_rows ||x_new - x_old||^2 (caller zeroes) */
    int32_t *d_status;       /* [1] 0, or 1 + first row whose system was not PD (caller zeroes) */
    int32_t vals_uniform;    /* 1 when every d_vals entry equals uniform_val (implicit feedback without
                                ratings): lets the Gram run on the tensor cores as v * M^T M */
    float uniform_val;
    /* Cooperative cancel (the role of CancelAdapter, src/accel/als/implicit.rs:72-73, tasks/mod.rs:62-106):
     * optional device flag, read (uncached) every time a CTA fetches work; once non-zero no further rows
     * are started — rows already solved keep their new values, the rest their old ones.  Progress =
     * *d_work_counter (groups of rows handed out so far), readable from another stream while the kernel runs. */
    const int32_t *d_cancel;
} lk_als_args;

LK_API int lk_als_half_epoch(const lk_als_args *args, void *stream);

/*
 * OtOr = O^T O + reg*I (k x k, f32), the role of _implicit_otor
 * (als/_implicit.py:177-184); optionally also writes the bf16 copy of O used by
 * the bf16-gather mode in the same pass.  d_scratch: [lk_als_otor_scratch_floats(k)].
 */
LK_API int64_t lk_als_otor_scratch_floats(int32_t k);
LK_API int lk_als_otor(const float *d_other, int64_t n_other, int32_t k, float reg, float *d_otor,
                void *d_other_bf16_or_null, float *d_scratch, void *stream);

/* ------------------------------------------------------------------------- */
/* item-kNN build                                                             */
/* ------------------------------------------------------------------------- */

typedef struct lk_knn_geom {
    int32_t n_users, n_items;
    int32_t warps;       /* warps per CTA (one accumulator sub-tile each) */
    int32_t tile_cols;   /* columns per warp sub-tile */
    int32_t n_halves;    /* column blocks per item row (CTA passes) */
    int32_t n_subtiles;  /* n_halves * warps */
    int32_t smem_bytes;  /* dynamic shared memory per CTA */
    int32_t ctas_per_sm;
} lk_knn_geom;

/* Choose the accumulator tiling for n_items columns on the current device. */
LK_API int lk_knn_geometry(int32_t n_users, int32_t n_items, lk_knn_geom *geom);

/* d_tile_ptr [n_users * (n_subtiles+1)]: for each user row of UI, the position of the
 * first column >= s*tile_cols (s = 0..n_subtiles). */
LK_API int lk_knn_tile_pointers(const lk_knn_geom *geom, const int32_t *d_ui_indptr,
                         const int32_t *d_ui_cols, int32_t *d_tile_ptr, void *stream);

/* d_cost [n_items] (int64): sum over the item's users of their row length —
 * the number of products sim_row does (item_train.rs:112-130); used to order
 * work longest-first and to shard rows across GPUs. */
LK_API int lk_knn_row_cost(const lk_knn_geom *geom, const int32_t *d_ui_indptr, const int32_t *d_iu_indptr,
                    const int32_t *d_iu_cols, int64_t *d_cost, void *stream);

typedef struct lk_knn_build_args {
    lk_knn_geom geom;
    const int32_t *d_ui_indptr, *d_ui_cols; const float *d_ui_vals; /* users x items */
    const int32_t *d_iu_indptr, *d_iu_cols; const float *d_iu_vals; /* items x users */
    const int32_t *d_tile_ptr;
    /* Work units.  d_units [n_units * 4] = {item, half, piece, n_pieces} stored item-major (an
     * item's units are d_unit_ptr[item] .. d_unit_ptr[item+1], halves and pieces ascending);
     * n_pieces in {1, 2, 4, 8} cuts the (item, half) unit of a very expensive item into column
     * slices so that several CTAs share it (only with save_nbrs > 0; the unbounded build needs
     * n_pieces == 1).  d_sched [n_work]: the unit ids to process, most expensive first — the
     * rows of a subset of items (item-sharded build) are produced by listing only their units. */
    const int32_t *d_units;
    const int32_t *d_unit_ptr; /* [n_items + 1] */
    int32_t max_units_per_item;
    const int32_t *d_sched;
    int64_t n_work;
    float min_sim;           /* keep dots >= min_sim (item_train.rs:133-137) */
    int32_t save_nbrs;       /* > 0: keep top-K per row (item_train.rs:140-147); <= 0: unbounded */
    /* truncated mode: per-unit partial lists, then merged */
    int32_t *d_part_cols;    /* [n_units * K] */
    float *d_part_vals;      /* [n_units * K] */
    int32_t *d_part_cnt;     /* [n_units] */
    /* unbounded mode: bump-allocated candidate pool */
    int32_t *d_pool_cols; float *d_pool_vals; int64_t pool_capacity;
    int64_t *d_pool_off;     /* [n_units] offsets into the pool */
    unsigned long long *d_pool_cursor; /* [1] zeroed by the caller */
    int32_t *d_tie_scratch;  /* [grid * half_cols * 3] per-CTA scratch for tie resolution */
    int32_t *d_work_counter; /* [1] zeroed by the call; = work units handed out so far (progress) */
    int32_t *d_status;       /* [1] 0 ok; 1 pool overflow; 2 NaN similarity */
    const int32_t *d_cancel; /* optional device flag (see lk_als_args.d_cancel): non-zero stops the hand-out of work */
} lk_knn_build_args;

LK_API int64_t lk_knn_tie_scratch_ints(const lk_knn_geom *geom);
LK_API int lk_knn_build(const lk_knn_build_args *args, void *stream);

/* Merge the per-half partial lists of the truncated build into fixed-width rows
 * sorted by column: out_cols/out_vals [n_items*K], out_cnt [n_items]. Tie-breaks
 * follow the reference's stable sort over first-touch order
 * (sim desc, first common user asc, column asc). */
LK_API int lk_knn_merge_topk(const lk_knn_build_args *args, int32_t *d_out_cols, float *d_out_vals,
                      int32_t *d_out_cnt, void *stream);

/* Unbounded mode: gather pool segments into CSR order given row offsets
 * d_out_indptr [n_items+1] (int64, exclusive scan of the per-row counts). */
LK_API int lk_knn_pool_to_csr(const lk_knn_build_args *args, const int64_t *d_out_indptr,
                       int32_t *d_out_cols, float *d_out_vals, void *stream);

/* ------------------------------------------------------------------------- */
/* user-kNN neighbour search (batched)                                        */
/* ------------------------------------------------------------------------- */

/*
 * The neighbour step of UserKNNScorer (src/lenskit/knn/user.py:189-214): for a batch of sparse query
 * vectors x_q, the users v with sim(q, v) = sum over the query's items i, ASCENDING, of VT[i,v] * x_q[i]
 * >= min_sim and v != self(q), in ascending v, with (float)sim as the weight.  VT is the item-major copy
 * of the f64 user_vectors matrix.  Every sum is accumulated in f64 in ascending item order with an
 * unfused multiply and add per step, starting from +0.0 — the order and rounding of SciPy's f64
 * `user_vectors @ x` (items outside the query only add +-0.0, which cannot change a nonzero sum), so the
 * neighbour set and the f32 weights are those of the reference bit for bit.  The comparison with min_sim
 * is made on the f64 sum.  See knn_user.cu.
 *
 * Geometry: the f64 accumulators of one query are tiled over the users; a CTA holds n_halves-th of them
 * (geom.warps sub-tiles of geom.tile_cols users).  In lk_knn_geom's own terms VT plays UI: its rows
 * (items) are geom.n_users and its columns (users) geom.n_items, so lk_knn_tile_pointers over VT with
 * this geometry gives d_tile_ptr [n_items * (n_subtiles+1)].  ctas_per_sm 0 = default (2).
 */
LK_API int lk_uknn_geometry(int32_t n_users, int32_t n_items, int32_t ctas_per_sm, lk_knn_geom *geom);

typedef struct lk_uknn_search_args {
    lk_knn_geom geom;                 /* lk_uknn_geometry */
    const int32_t *d_vt_indptr;       /* [n_items+1] VT: items x users */
    const int32_t *d_vt_users;        /* [nnz] users ascending within an item */
    const double *d_vt_vals;          /* [nnz] user_vectors values (f64) */
    const int32_t *d_tile_ptr;        /* lk_knn_tile_pointers(geom, d_vt_indptr, d_vt_users) */
    int32_t n_queries;                /* B; B * geom.n_halves < 2^31 */
    const int64_t *d_q_begin;         /* [B] query q is entries [d_q_begin[q], d_q_end[q]) of d_q_items / d_q_vals */
    const int64_t *d_q_end;           /* [B] (e.g. rows of the row-major user_vectors, or an uploaded CSR) */
    const int32_t *d_q_items;         /* items strictly ascending within a query, in [0, n_items) */
    const double *d_q_vals;           /* f64 query values */
    const int32_t *d_q_self;          /* [B] user excluded from query q's neighbours, or -1; NULL = none */
    double min_sim;                   /* keep sim >= min_sim, compared in f64; > 0 */
    /* work units: unit id = q * n_halves + h (query q, user tile h); d_sched [n_work] lists the units to
     * process, most expensive first.  Units not listed produce nothing (their d_part_cnt stays as given). */
    const int32_t *d_sched;
    int64_t n_work;
    /* survivors, bump-allocated per unit in tile order */
    int32_t *d_pool_rows;             /* [pool_capacity] neighbour user */
    float *d_pool_sims;               /* [pool_capacity] (float)sim */
    int64_t pool_capacity;            /* e.g. sum over q of min(lk_uknn_query_cost(q), n_users) */
    int64_t *d_pool_off;              /* [B * n_halves] offset of the unit's segment */
    int32_t *d_part_cnt;              /* [B * n_halves] length of the unit's segment */
    unsigned long long *d_pool_cursor; /* [1] zeroed by the call */
    int32_t *d_work_counter;          /* [1] zeroed by the call */
    int32_t *d_status;                /* [1] zeroed by the call; 1 = pool overflow (then nothing is usable) */
} lk_uknn_search_args;

/* d_cost [B] (int64): sum over the query's items of |VT row| — the products of its search. */
LK_API int lk_uknn_query_cost(const lk_uknn_search_args *args, int64_t *d_cost, void *stream);
LK_API int lk_uknn_search(const lk_uknn_search_args *args, void *stream);
/* Gather the pool segments into CSR: d_out_indptr [B+1] (int64, exclusive scan of the per-query sums of
 * d_part_cnt) -> d_out_rows / d_out_sims, rows ascending within a query.  This is the neighbour-list layout
 * lk_knn_score_batch takes in user mode (d_ref_indptr / d_ref_items / d_ref_vals). */
LK_API int lk_uknn_pool_to_csr(const lk_uknn_search_args *args, const int64_t *d_out_indptr, int32_t *d_out_rows,
                               float *d_out_sims, void *stream);

/* ------------------------------------------------------------------------- */
/* item-kNN input preparation (SURVEY.md 8f N4)                               */
/* ------------------------------------------------------------------------- */

/*
 * Mean-centre (centre != 0: explicit feedback) and unit-L2-normalise the item columns of the rating
 * matrix — the host stage of ItemKNNScorer.train, src/lenskit/knn/item.py:202-228
 * (_center_ratings, _normalize_rows), reproduced bit for bit (NumPy's pairwise float32 / float64
 * summation order, float64 norm and reciprocal, float32 result; see prep.cu).
 * d_indptr [n_cols+1] / d_vals [nnz]: the ratings in CSC order (items major, users ascending);
 * d_means [n_cols] (may be NULL) receives the float32 item means (0 for empty items and when not
 * centring); d_out [nnz] the normalised values in the same order — together with the user
 * indices this is the IU matrix compute_similarities takes, and its transpose is UI.
 */
LK_API int lk_knn_prep_columns(const int32_t *d_indptr, const float *d_vals, int32_t n_cols, int32_t centre,
                               float *d_means, float *d_out, void *stream);

/* ------------------------------------------------------------------------- */
/* item-kNN scoring (batched over queries)                                    */
/* ------------------------------------------------------------------------- */

typedef struct lk_knn_score_args {
    int32_t n_items;
    const int64_t *d_sim_indptr; /* [n_items+1] (LargeList offsets, item_score.rs:113-118) */
    const int32_t *d_sim_cols; const float *d_sim_vals; /* rows sorted by column */
    int32_t n_queries;
    const int64_t *d_ref_indptr; /* [n_queries+1] query histories as CSR, in history order */
    const int32_t *d_ref_items;  /* negative = null, skipped */
    const float *d_ref_vals;     /* mean-centred ratings, or NULL for implicit feedback */
    const int64_t *d_tgt_indptr; /* [n_queries+1] */
    const int32_t *d_tgt_items;  /* negative = null -> score NaN, count -1 */
    int32_t max_nbrs, min_nbrs;
    int32_t *d_slotmap;          /* [slotmap_warps * n_items], all -1 on entry and on exit */
    int64_t slotmap_warps;       /* warps that work on the batch, one slot-map row each: 1..lk_knn_score_warps()
                                    (more is not used); min(n_queries, lk_knn_score_warps()) is enough */
    int32_t *d_list_off, *d_list_cur; /* [n_targets] each: a target's contribution-list offset and fill cursor */
    int32_t *d_list_cnt;         /* [n_targets]: contributions per target */
    float *d_scores;             /* [n_targets] NaN = null (Arrow null in the reference) */
    int32_t *d_counts;           /* [n_targets] -1 = null */
    int32_t *d_work_counter;     /* [1] zeroed by the call */
    int32_t *d_status;           /* [1] 0 ok; 2 NaN similarity */
    /* Contribution pool (required): per-target contribution lists are built in parallel, sorted by
     * history position and replayed through the accumulator.  pool_entries 16-byte entries, at least
     * the number of (reference item, similarity-row entry) pairs of the whole batch:
     * sum over valid d_ref_items r of (d_sim_indptr[r+1] - d_sim_indptr[r]); d_pool_cursor [1]
     * is zeroed by the call.  Status 3 = pool too small. */
    void *d_pool;
    int64_t pool_entries;
    unsigned long long *d_pool_cursor;
    /* 0: item-kNN (above).  1: user-kNN scoring, src/accel/knn/user_score.rs:21-98 — the same
     * accumulators with the roles of the two operands swapped: the "history" of a query is its
     * neighbour list (d_ref_items = neighbour user rows, d_ref_vals = their similarities = the
     * WEIGHTS, required), the matrix is the users x items rating matrix (d_sim_* = its CSR;
     * d_sim_vals = centred ratings = the VALUES, NULL for implicit feedback), n_items = its number
     * of columns, and a row index is valid in [0, n_matrix_rows). */
    int32_t user_mode;
    int32_t n_matrix_rows;       /* user mode: rows of the rating matrix (item mode: unused, = n_items) */
    /* Dense mode — d_tgt_indptr == NULL and d_tgt_items == NULL: every query is scored against ALL
     * items in index order; d_scores / d_counts are [n_queries * n_items] and written exactly once, d_list_cnt
     * is not used.  A CTA handles a query and keeps its state per CTA: d_slotmap provides one n_items row per
     * CTA (slotmap_warps >= lk_knn_score_dense_ctas()) that must be all ZERO on entry and is left all zero
     * (item -> touched-target number), d_list_off / d_list_cur one n_items row per CTA each
     * ([min(n_queries, lk_knn_score_dense_ctas()) * n_items]: list offsets / cursors by touched-target number). */
} lk_knn_score_args;

/* largest number of warps the scoring grid runs (one slotmap row each) */
LK_API int64_t lk_knn_score_warps(void);
/* number of CTAs of the dense (all-items) scoring grid: one n_items row of d_slotmap each */
LK_API int64_t lk_knn_score_dense_ctas(void);
LK_API int lk_knn_score_batch(const lk_knn_score_args *args, void *stream);

/*
 * Batched top-n recommendation from the kNN scorers (dense mode with ranking, knn_score.cu): for every query,
 * the reference's composition of TrainingItemsCandidateSelector, the scorer and TopNRanker,
 *     cands = all items ascending, minus the query's excluded items;  il = scorer(query, cands);
 *     top   = il[argtopn(il.scores, n)]
 * with the final score of an item = (accumulator score + d_item_offset[item]) + d_query_offset[q], f32 adds
 * (NaN stays NaN).  The selection replays argtopn's heap (see lk_topn_columns), so ties are cut and ordered
 * exactly as there.  `score` is an lk_knn_score_args in dense mode (d_tgt_indptr == d_tgt_items == NULL) with
 * the same layout rules; its d_scores / d_counts are not used.  Per query q, n entries at q*n:
 *   d_out_idx   item number of rank t, -1 beyond the count
 *   d_out_val   its final score, NaN beyond the count
 *   d_out_nbrs  its accumulator length (the scorer's nbr_counts), 0 beyond the count
 *   d_out_cnt   [q] = min(n, number of candidates with a non-NaN score)
 * d_spill: one n_items int32 row per CTA ([lk_knn_score_dense_ctas() * n_items]) for the touched-target list
 * of a query that touches more targets than the CTA keeps in shared memory; any content on entry.
 * Statuses as lk_knn_score_batch (2 NaN similarity, 3 pool too small).
 */
typedef struct lk_knn_rank_args {
    int32_t n;                     /* 1..lk_topn_max() */
    const float *d_item_offset;    /* [n_items] or NULL */
    const float *d_query_offset;   /* [n_queries] or NULL */
    const int64_t *d_excl_indptr;  /* [n_queries+1] or NULL: items never recommended to the query */
    const int32_t *d_excl_items;   /* any order, repeats allowed, negative skipped */
    int32_t *d_spill;              /* per-CTA touched-target spill rows */
    int32_t *d_out_idx; float *d_out_val; int32_t *d_out_nbrs; /* [n_queries * n] */
    int32_t *d_out_cnt;            /* [n_queries] */
} lk_knn_rank_args;
LK_API int lk_knn_recommend_batch(const lk_knn_score_args *score, const lk_knn_rank_args *rank, void *stream);

/* ------------------------------------------------------------------------
 * Batched ALS scoring and top-n recommendation (als_recommend.cu).  For query b with embedding x_b
 * (d_queries row b) and item i (d_items row i), the score is one fp32 FMA chain in ascending d,
 *     s = +0.0f;  for d = 0 .. k-1:  s = fmaf(Q[i,d], x_b[d], s)
 * then s = s + d_item_offset[i] and s = s + d_query_offset[b] (f32 adds, each only when the pointer is set).
 *   n == 0   score mode: d_scores[i * n_queries + b] = s (item-major, the layout of Q . X^T);
 *   n >= 1   rank mode (n <= lk_topn_max()): for every query, argtopn over its candidates (all items ascending,
 *            minus d_excl_items[d_excl_indptr[b] .. d_excl_indptr[b+1]]), ties included, written like
 *            lk_topn_columns' outputs but query-major:
 *              d_out_idx[b*n + t]  item number of rank t, -1 beyond the count
 *              d_out_val[b*n + t]  its score, NaN beyond the count
 *              d_out_cnt[b]        the number of candidates with a non-NaN score, at most n
 *            The excluded items must be ASCENDING within each query; repeats and negative numbers are allowed
 *            (and skipped).  d_excl_indptr may be NULL (nothing excluded).  n > 128 keeps the heaps in
 *            d_workspace, lk_als_recommend_workspace_bytes(n_queries, n) bytes (NULL when that is 0).
 * k in 1..128; n_items < 2^31.  Both modes share the dot products, so argtopn over a score-mode column gives
 * the rank-mode list bit for bit.  The grid is one CTA per 64 queries sweeping every item: batch widely.
 * ---------------------------------------------------------------------- */
typedef struct lk_als_rec_args {
    int64_t n_items;
    int32_t k;                      /* 1..128 */
    int32_t n_queries;
    const float *d_items;           /* Q [n_items][k], row-major */
    const float *d_queries;         /* X [n_queries][k], row-major */
    const float *d_item_offset;     /* [n_items] or NULL */
    const float *d_query_offset;    /* [n_queries] or NULL */
    int32_t n;                      /* 0: score mode; 1..lk_topn_max(): rank mode */
    float *d_scores;                /* score mode: [n_items][n_queries] */
    const int64_t *d_excl_indptr;   /* rank mode: [n_queries+1] or NULL */
    const int32_t *d_excl_items;    /* ascending within a query, repeats allowed, negative skipped */
    void *d_workspace;              /* lk_als_recommend_workspace_bytes(n_queries, n) bytes */
    int32_t *d_out_idx; float *d_out_val; /* [n_queries * n] */
    int32_t *d_out_cnt;             /* [n_queries] */
} lk_als_rec_args;
LK_API int64_t lk_als_recommend_workspace_bytes(int32_t n_queries, int32_t n);
LK_API int lk_als_recommend_batch(const lk_als_rec_args *args, void *stream);

/* ------------------------------------------------------------------------
 * Batched top-N (SURVEY.md §8f N2: the step after the scorer)
 *
 * Replaces `_accel.data.argtopn` (src/accel/data/sorting.rs:131-170; the selection
 * behind ItemList.top_n, src/lenskit/data/_items.py:942-998, and TopNRanker,
 * src/lenskit/basic/topn.py:32-69) for every column of a row-major score matrix
 * d_scores[n_rows][ld] (rows = items, columns = score vectors, e.g. Q . X^T).
 * Column c gets the indices of its n largest non-NaN scores in the reference's
 * order — the kernel replays the reference's indirect min-heap
 * (src/accel/indirect/heap.rs), so ties are cut and ordered exactly as there:
 *   d_out_idx[c*n + t]  item index of rank t, -1 beyond the column's count
 *   d_out_val[c*n + t]  its score (NaN beyond the count); may be NULL
 *   d_out_cnt[c]        min(n, number of non-NaN scores in the column)
 * n in 1..lk_topn_max(); n_rows < 2^31.
 * ---------------------------------------------------------------------- */
LK_API int lk_topn_max(void);
LK_API int lk_topn_columns(const float *d_scores, int64_t n_rows, int64_t n_cols, int64_t ld, int32_t n,
                           int32_t *d_out_idx, float *d_out_val, int32_t *d_out_cnt, void *stream);

/* ------------------------------------------------------------------------
 * Co-occurrence counting (cooc.cu): the counts of `_accel.data.count_cooc` / `dense_cooc`
 * (src/accel/data/cooc.rs:185-214, pairs/symmetric.rs, pairs/dense.rs) and the association matrix of
 * AssociationScorer.train (src/lenskit/knn/association.py:91-130).
 *
 * The groups play the users of the item-kNN build: GI is the groups x items CSR (a group's items ascending,
 * repeated items kept), IG its transpose with one entry per occurrence.  Row i of the result is
 *     C[i][j] = sum over the occurrences of i in a group g of the occurrences of j in g  (= sum_g #i * #j)
 * over the columns j > i (full_rows == 0, the strict upper triangle) or j != i (full_rows == 1).  The diagonal
 * sum_g #i (#i + 1) / 2 comes from lk_cooc_diagonal.  Work units are (item, column tile):
 * unit = item * geom.n_halves + h; units not listed in d_sched produce nothing (their d_part_cnt stays as
 * given, so the caller zeroes it).  Survivors (non-zero counts) go to a bump-allocated pool in column order per
 * unit; lk_cooc_pool_to_csr gathers them into a row-sorted CSR with int64 offsets.
 *   method LK_COOC_COUNT: pool values are the int32 counts;
 *   LK_ASSOC_PROBABILITY / LK_ASSOC_LIFT (full_rows == 1): the f32 association value of entry (r, c),
 *     v = f32(f64(f32(count)) / (f64(cnt[r]) + damping));  lift: v = f32(v * f32(n_groups)),
 *     v = f32(f64(v) / (f64(cnt[c]) + damping))          (cnt = d_item_count, n_groups = geom.n_users)
 * Every count of a row is at most the row's cost (lk_cooc_row_cost); the caller passes the largest cost in
 * max_row_cost and a value of 2^31 or more returns LK_ERR_UNSUPPORTED instead of wrapping.
 * Statuses: 1 = pool too small (nothing is usable; never a truncated result).
 * ---------------------------------------------------------------------- */
#define LK_COOC_COUNT 0
#define LK_ASSOC_PROBABILITY 1
#define LK_ASSOC_LIFT 2

/* Accumulator tiling for n_cols columns over the rows of an n_rows-row CSR whose tile pointers are taken
 * (groups for counting, items for association scoring). */
LK_API int lk_cooc_geometry(int32_t n_rows, int32_t n_cols, lk_knn_geom *geom);

typedef struct lk_cooc_args {
    lk_knn_geom geom;                  /* lk_cooc_geometry(n_groups, n_items) */
    const int32_t *d_gi_indptr;        /* [n_groups+1] */
    const int32_t *d_gi_items;         /* ascending within a group, repeats kept */
    const int32_t *d_ig_indptr;        /* [n_items+1] */
    const int32_t *d_ig_groups;        /* one entry per occurrence */
    const int32_t *d_tile_ptr;         /* lk_knn_tile_pointers(geom, d_gi_indptr, d_gi_items) */
    int32_t full_rows;                 /* 0: columns > row; 1: every column but the row */
    int32_t method;                    /* LK_COOC_COUNT or LK_ASSOC_* */
    const int32_t *d_item_count;       /* [n_items] per-item interaction counts (LK_ASSOC_*) */
    double damping;                    /* >= 0 */
    int64_t max_row_cost;              /* largest lk_cooc_row_cost of a scheduled row */
    const int32_t *d_sched;            /* [n_work] unit ids, most expensive first */
    int64_t n_work;
    int32_t *d_pool_cols;              /* [pool_capacity] */
    void *d_pool_vals;                 /* [pool_capacity] 32-bit: int32 counts or f32 values */
    int64_t pool_capacity;
    int64_t *d_pool_off;               /* [n_items * n_halves] */
    int32_t *d_part_cnt;               /* [n_items * n_halves] */
    unsigned long long *d_pool_cursor; /* [1] zeroed by the call */
    int32_t *d_work_counter;           /* [1] zeroed by the call; = units handed out so far (progress) */
    int32_t *d_status;                 /* [1] zeroed by the call */
    const int32_t *d_cancel;           /* optional device flag (see lk_als_args.d_cancel) */
} lk_cooc_args;

/* d_cost [n_items] (int64): the pair updates of each row, sum over its occurrences of the group's columns
 * that the row counts (columns > item, or the whole group with full_rows). */
LK_API int lk_cooc_row_cost(const lk_cooc_args *args, int64_t *d_cost, void *stream);
LK_API int lk_cooc_count(const lk_cooc_args *args, void *stream);
/* d_out_indptr [n_items+1]: exclusive scan of the per-item sums of d_part_cnt; d_out_vals 32-bit words */
LK_API int lk_cooc_pool_to_csr(const lk_cooc_args *args, const int64_t *d_out_indptr, int32_t *d_out_cols,
                               void *d_out_vals, void *stream);
/* d_diag [n_items] (int64, zeroed by the caller) += sum over groups of #i (#i + 1) / 2 */
LK_API int lk_cooc_diagonal(const lk_cooc_args *args, int64_t *d_diag, void *stream);
/* Dense sink of dense_cooc: d_out [n_items][n_items] f32 (zeroed by the caller) gets f32(count) of every entry
 * of the strict-upper-triangle CSR at (i, j) and (j, i), and f32(d_diag[i]) at (i, i) when d_diag is set. */
LK_API int lk_cooc_dense(int32_t n_items, const int64_t *d_indptr, const int32_t *d_cols, const int32_t *d_counts,
                         const int64_t *d_diag, float *d_out, void *stream);

/* ------------------------------------------------------------------------
 * Association scoring (cooc.cu): AssociationScorer.__call__ (association.py:132-163) batched, and its
 * composition with TrainingItemsCandidateSelector and TopNRanker.  For query q with reference rows
 * r_0 .. r_{R-1} (d_ref_items in query order, repeats kept, all in [0, n_items)) and item c:
 *   agg 0 (mean, max_nbrs = None):  s = +0.0f;  for t = 0 .. R-1: s = s + A[r_t, c]  (f32 adds in query order,
 *                                   absent entries add nothing);  score = f32(f64(s) / f64(R))
 *   agg 1 (max, max_nbrs = 1):      score = max over t of A[r_t, c], absent entries 0; the max starts at +0.0f,
 *                                   so A must be non-negative (as training makes it; NaN entries are outside
 *                                   the contract: fmaxf drops them where np.max would propagate them)
 *   agg 2 (sum, SLIMScorer):        s as for agg 0, score = s (no divide)
 *   R == 0: every score is NaN (agg 0, 1; rank mode recommends nothing), +0.0 (agg 2; rank mode ranks the zeros).
 * A is the association CSR (int64 offsets, rows sorted by column); d_tile_ptr [n_items * (n_subtiles+1)] holds,
 * for each row and s = 0..n_subtiles, the position of its first column >= s * tile_cols RELATIVE to the row
 * start (lk_assoc_tile_pointers).
 *   n == 0  score mode: d_scores [n_queries][n_items].
 *   n >= 1  rank mode (n <= lk_topn_max()): argtopn over every item ascending minus the query's excluded items
 *           (ascending within a query, repeats and negative numbers skipped), ties included; a NaN score (+inf
 *           and -inf at one column of two reference rows) is never offered, as argtopn skips it; outputs as
 *           lk_als_recommend_batch's rank mode.
 * n_queries * geom.n_halves < 2^31.
 * ---------------------------------------------------------------------- */
LK_API int lk_assoc_tile_pointers(const lk_knn_geom *geom, const int64_t *d_indptr, const int32_t *d_cols,
                                  int32_t *d_tile_ptr, void *stream);

typedef struct lk_assoc_score_args {
    lk_knn_geom geom;                  /* lk_cooc_geometry(n_items, n_items) */
    const int64_t *d_indptr;           /* [n_items+1] */
    const int32_t *d_cols;
    const float *d_vals;
    const int32_t *d_tile_ptr;
    int32_t n_queries;
    int32_t agg;                       /* 0 mean, 1 max, 2 sum */
    const int64_t *d_ref_indptr;       /* [n_queries+1] */
    const int32_t *d_ref_items;
    int32_t n;                         /* 0: score mode; 1..lk_topn_max(): rank mode */
    float *d_scores;                   /* score mode: [n_queries][n_items] */
    const int64_t *d_excl_indptr;      /* rank mode: [n_queries+1] or NULL */
    const int32_t *d_excl_items;
    int32_t *d_out_idx; float *d_out_val; /* rank mode: [n_queries * n] */
    int32_t *d_out_cnt;                /* rank mode: [n_queries] */
} lk_assoc_score_args;

LK_API int lk_assoc_score_batch(const lk_assoc_score_args *args, void *stream);

/* ------------------------------------------------------------------------
 * EASE scoring (ease.cu): EASEScorer.__call__ (src/lenskit/knn/ease.py), `q_vec @ weights` with a 0/1 query
 * vector, batched, and its composition with TrainingItemsCandidateSelector and TopNRanker.  W is the dense
 * f32 weight matrix [n_items][n_items], row-major.  For query q with history H_q = d_hist_items[
 * d_hist_indptr[q] .. d_hist_indptr[q+1]) (ascending, no repeats, all in [0, n_items)) and item j:
 *     s = +0.0f;  for h in H_q in order: s = s + W[h][j]      (f32 adds, round to nearest)
 *   H_q empty: every score is NaN (score mode), an empty list (rank mode).
 *   n == 0  score mode: d_scores [n_queries][n_items].
 *   n >= 1  rank mode (n <= lk_topn_max()): argtopn over every item ascending minus the query's excluded items
 *           (ascending within a query), ties included; outputs as lk_assoc_score_batch's rank mode.
 * n_queries * ceil(n_items / 1024) < 2^31.
 * ---------------------------------------------------------------------- */
typedef struct lk_ease_score_args {
    int32_t n_items;
    const float *d_w;                  /* [n_items][n_items] */
    int32_t n_queries;
    const int64_t *d_hist_indptr;      /* [n_queries+1] */
    const int32_t *d_hist_items;
    int32_t n;                         /* 0: score mode; 1..lk_topn_max(): rank mode */
    float *d_scores;                   /* score mode: [n_queries][n_items] */
    const int64_t *d_excl_indptr;      /* rank mode: [n_queries+1] or NULL */
    const int32_t *d_excl_items;
    int32_t *d_out_idx; float *d_out_val; /* rank mode: [n_queries * n] */
    int32_t *d_out_cnt;                /* rank mode: [n_queries] */
} lk_ease_score_args;

LK_API int lk_ease_score_batch(const lk_ease_score_args *args, void *stream);

/* ------------------------------------------------------------------------
 * SLIM training (slim.cu): `_accel.slim.train_slim` (src/accel/slim/mod.rs:57-93), one weight column per target
 * item i, rows of the result in item order.  UI (users x items) and IU (items x users) are CSR structures walked in
 * stored order (UI rows need not be sorted; an IU row must not repeat a user).  For target i with users U_i:
 *   resid[u] = 1 on U_i, 0 elsewhere; active = the items j != i of the UI rows of U_i in first-encounter order,
 *   pc[j] their encounter counts; with 0 <= max_nbrs < |active|, active is stably sorted by the f64 key
 *   -pc[j] / (sqrt(|U_i|) * sqrt(|U_j|)) and cut to max_nbrs.  Up to max_iters rounds over active, each j:
 *   upd = +0.0f, upd += (resid[u] + W[j]) over U_j in order; new = upd >= l1 ? (upd - l1) / (f32(|U_j|) + l2) : 0;
 *   diff = new - W[j]; W[j] = new; resid[u] -= diff over U_j; the round stops CD when max |diff| <= 1e-3f.
 *   All f32 operations rounded to nearest, none contracted.  Row i: every j ascending with W[j] >= 1e-12f.
 * Work units are target items (d_sched, a permutation of a subset of the items, most expensive first: see
 * lk_cooc_row_cost with full rows over GI = UI, IG = IU); rows not listed keep the d_part_cnt given (zeroed by the
 * caller).  Each warp of the grid owns lk_slim_workspace_bytes / warps of d_workspace, which must be zero before
 * the first call and is zero again after every call.  Survivors go to a bump-allocated pool (one segment per row);
 * lk_slim_pool_to_csr gathers them into a row-sorted CSR with int64 offsets.  d_work_counter counts the rows handed
 * out (progress); the optional d_cancel flag stops handing out rows.
 * Statuses: 1 = pool too small (nothing is usable; never a truncated result).
 * ---------------------------------------------------------------------- */
typedef struct lk_slim_args {
    int32_t n_users, n_items;
    const int32_t *d_ui_indptr;        /* [n_users+1] */
    const int32_t *d_ui_cols;          /* items, in [0, n_items) */
    const int32_t *d_iu_indptr;        /* [n_items+1] */
    const int32_t *d_iu_cols;          /* users, in [0, n_users) */
    float l1_reg, l2_reg;
    int32_t max_iters;                 /* >= 0 */
    int32_t max_nbrs;                  /* fsSLIM neighbours, or -1 (SLIM) */
    const int32_t *d_sched;            /* [n_work] target items */
    int64_t n_work;                    /* <= n_items */
    void *d_workspace;
    int64_t workspace_bytes;
    int32_t *d_pool_cols;              /* [pool_capacity] */
    float *d_pool_vals;                /* [pool_capacity] */
    int64_t pool_capacity;
    int64_t *d_pool_off;               /* [n_items] */
    int32_t *d_part_cnt;               /* [n_items] */
    unsigned long long *d_pool_cursor; /* [1] zeroed by the call */
    int32_t *d_work_counter;           /* [1] zeroed by the call */
    int32_t *d_status;                 /* [1] zeroed by the call */
    const int32_t *d_cancel;           /* optional device flag (see lk_als_args.d_cancel) */
} lk_slim_args;

/* *bytes: the workspace lk_slim_train needs for n_work rows on the current device */
LK_API int lk_slim_workspace_bytes(int32_t n_users, int32_t n_items, int64_t n_work, int64_t *bytes);
LK_API int lk_slim_train(const lk_slim_args *args, void *stream);
/* d_out_indptr [n_items+1]: exclusive scan of d_part_cnt */
LK_API int lk_slim_pool_to_csr(const lk_slim_args *args, const int64_t *d_out_indptr, int32_t *d_out_cols,
                               float *d_out_vals, void *stream);

/* ------------------------------------------------------------------------
 * FlexMF (flexmf.cu): gradient-trained matrix factorisation with logistic or pairwise (BPR) loss,
 * FlexMFImplicitTrainer (src/lenskit/flexmf/_implicit.py, _training.py, _model.py), or with squared error on
 * centred ratings, FlexMFExplicitTrainer (src/lenskit/flexmf/_explicit.py).  Score of (u, i):
 * s = ub[u] + ib[i] + <U[u], I[i]>, an absent bias vector counting as 0.
 *
 * Negative sampling.  For sample g of d_rows (a user), step = step0 + g / batch_size, pos = g % batch_size, and
 * rep < n: draw columns attempt = 0, 1, ... and keep the first that is not a column of the user's CSR row, or the
 * draw of attempt == max_attempts whatever it is (the procedure of sampling.rs:38-58; the stream is this
 * library's own).  With all arithmetic in uint64, wrapping:
 *     mix(x):  x ^= x >> 30;  x *= 0xbf58476d1ce4e5b9;  x ^= x >> 27;  x *= 0x94d049bb133111eb;  x ^= x >> 31
 *     G = 0x9e3779b97f4a7c15
 *     h = mix(seed + G * (step + 1));  h = mix(h + G * (pos + 1));  h = mix(h + G * ((rep << 32) + attempt + 1))
 *     draw(m) = ((h >> 32) * m) >> 32                      in [0, m); no value is more than m / 2^32 (relative)
 *                                                          more likely than another
 *   uniform: column = draw(n_items);  popular: column = d_coo_items[draw(nnz)], a uniformly drawn training
 *   interaction's item.  d_out [n_samples][n].  CSR columns ascending within a row (membership is a binary search).
 * ---------------------------------------------------------------------- */
typedef struct lk_flexmf_sample_args {
    int32_t n_users, n_items;
    const int32_t *d_ui_indptr;        /* [n_users+1] */
    const int32_t *d_ui_cols;          /* items, ascending within a row */
    const int32_t *d_coo_items;        /* [nnz] item of every training interaction (popular only) */
    int64_t nnz;                       /* < 2^32 */
    const int32_t *d_rows;             /* [n_samples] users */
    int64_t n_samples;
    int32_t batch_size;                /* samples per step (>= 1) */
    int32_t n;                         /* negatives per sample (>= 1) */
    int32_t max_attempts;              /* rejected draws before one is kept regardless (the reference: 10) */
    int32_t popular;                   /* 0 uniform, 1 popularity-weighted */
    uint64_t seed;
    int64_t step0;                     /* step number of sample 0 */
    int32_t *d_out;                    /* [n_samples][n] */
} lk_flexmf_sample_args;

LK_API int lk_flexmf_sample_negatives(const lk_flexmf_sample_args *args, void *stream);

#define LK_FLEXMF_LOGISTIC 0
#define LK_FLEXMF_PAIRWISE 1
#define LK_FLEXMF_MSE 2        /* rating regression: n_neg = 0 and d_ratings required */
#define LK_FLEXMF_REG_NONE 0   /* torch.optim.SparseAdam */
#define LK_FLEXMF_REG_L2 1     /* explicit norm term in the loss, SparseAdam */
#define LK_FLEXMF_REG_ADAMW 2  /* torch.optim.AdamW(weight_decay = regularization) over every parameter */

/*
 * The occurrences of one side's rows (users, or items) in the batches, grouped by the caller.  Users occur once per
 * sample (entry: the sample's position b in its batch); items once per (sample, slot) with slot 0 the positive and
 * 1..n the negatives (entry: b * (n + 1) + slot).  Entries are sorted by (step, row, entry) in d_occ; every maximal
 * run of one (step, row) is a "uniq", cut into "units" of at most 64 consecutive entries.  All indices are into the
 * arrays given, which may cover many steps; a step uses units [unit0, unit0 + n_units) and uniqs [uniq0, uniq0 + n_uniq).
 */
typedef struct lk_flexmf_groups {
    const int32_t *d_occ;
    const int64_t *d_unit_start;       /* [units + 1] offsets into d_occ */
    const int32_t *d_unit_uniq;        /* [units] the uniq a unit belongs to */
    const int32_t *d_uniq_row;         /* [uniqs] row number */
    const int32_t *d_uniq_unit;        /* [uniqs + 1] first unit of every uniq */
    int64_t unit0, uniq0;
    int32_t n_uniq;
    int64_t *d_mark;                   /* AdamW: [n_rows], zero before step 1; (step << 32 | uniq) of the last touch */
} lk_flexmf_groups;

/*
 * One minibatch step, in place: the loss of the batch as the reference defines it
 *   logistic: (sum_b -log sigma(s+_b) * positive_weight + sum_{b,r} -log sigma(-s-_{b,r})) / (B + B n)
 *   pairwise: mean over the B n pairs of -log sigma(s+_b - s-_{b,r})
 *   MSE:      mean_b (s_b - t_b)^2 with t = d_ratings (n_neg = 0: every sample has only its rated item, slot 0)
 *   LK_FLEXMF_REG_L2 adds regularization * 0.5 * (mean_b norm+ + mean_{b,r} norm-) to the logistic and pairwise
 *   losses and regularization * mean_b norm_b to MSE, norm = ub^2 + ib^2 + |U[u]| + |I[i]| (vector norms not
 *   squared; the gradient of |x| at x = 0 is 0).  Per occurrence in the batch, its gradient is
 *     user rows (every loss):            regularization / B * (U / |U|, 2 ub)
 *     item rows, logistic and pairwise:  0.5 regularization / B * (I / |I|, 2 ib) as the positive,
 *                                        0.5 regularization / (B n) * (I / |I|, 2 ib) as a negative
 *     item rows, MSE:                    regularization / B * (I / |I|, 2 ib), twice the implicit positive's
 *   MSE's d_loss is the squared error alone, without the norm term (the reference's train_batch returns that),
 * its gradient with every row's contributions added in a fixed order (ascending entry within a unit, a user's
 * items of one sample combined first, units of a row ascending), then the optimiser (betas, eps as given;
 * the host passes the scalars that depend on the step number):
 *   AdamW      every row:  w *= decay;  m += (g - m)(1 - beta1);  v = v beta2 + (1 - beta2) g^2;
 *                          w -= step_size * m / (sqrt(v) / bias2_sqrt + eps)     with step_size = lr / (1 - beta1^t)
 *   SparseAdam rows of the batch only:  m += (g - m)(1 - beta1);  v += (g^2 - v)(1 - beta2);
 *                          w -= step_size * m / (sqrt(v) + eps)     with step_size = lr sqrt(1 - beta2^t) / (1 - beta1^t)
 * d_loss[0] receives the batch loss (f32, summed in f64 in a fixed order).  No float atomics: the result is a pure
 * function of the arguments.  k <= lk_als_max_features().
 */
typedef struct lk_flexmf_step_args {
    int32_t n_users, n_items, k;
    int32_t batch;                     /* B: samples in this step */
    int32_t n_neg;                     /* n: >= 1, or 0 with MSE */
    int32_t loss;                      /* LK_FLEXMF_LOGISTIC / _PAIRWISE / _MSE */
    int32_t reg_method;                /* LK_FLEXMF_REG_* */
    float positive_weight, regularization;
    float decay;                       /* AdamW: 1 - lr * regularization */
    float one_minus_beta1, beta2, one_minus_beta2, eps;
    float step_size, bias2_sqrt;       /* see above; bias2_sqrt = sqrt(1 - beta2^t), AdamW only */
    int64_t step;                      /* t >= 1, below 2^31 */
    float *d_u_emb, *d_u_emb_m, *d_u_emb_v;    /* [n_users][k] parameters and the two moments */
    float *d_i_emb, *d_i_emb_m, *d_i_emb_v;    /* [n_items][k] */
    float *d_u_bias, *d_u_bias_m, *d_u_bias_v; /* [n_users] or all NULL */
    float *d_i_bias, *d_i_bias_m, *d_i_bias_v; /* [n_items] or all NULL */
    const int32_t *d_users;            /* [B] */
    const int32_t *d_pos;              /* [B] */
    const int32_t *d_neg;              /* [B][n]; unused (may be NULL) with MSE */
    lk_flexmf_groups u_groups, i_groups;
    int32_t n_u_units, n_i_units;
    void *d_workspace;
    int64_t workspace_bytes;           /* >= lk_flexmf_workspace_bytes(batch, n_neg, k) */
    float *d_loss;                     /* [1] */
    const float *d_ratings;            /* [B] targets t = r - mu, MSE only */
} lk_flexmf_step_args;

LK_API int lk_flexmf_workspace_bytes(int32_t batch, int32_t n_neg, int32_t k, int64_t *bytes);
LK_API int lk_flexmf_step(const lk_flexmf_step_args *args, void *stream);

/* ------------------------------------------------------------------------
 * Sparse x dense product (spmm.cu), the products of TruncatedSVD's randomized SVD (BiasedSVDScorer,
 * src/lenskit/sklearn/svd.py).  Y [n_rows][W] = A D with A a CSR [n_rows x n_src] and D [n_src][W] row-major:
 *     Y[r][c] = +0.0f;  for p in row r in stored order: Y[r][c] = Y[r][c] + val[p] * D[idx[p]][c]
 * with the product and the sum each rounded to nearest (never one FMA).  That is SciPy's f32 `A @ D` bit for bit;
 * `A.T @ D` and `D.T @ A` are the same walk over the transposed CSR (rows in ascending order inside a row).
 * d_order lists every row once, longest first: the order in which rows are handed to the warps.
 * ---------------------------------------------------------------------- */
typedef struct lk_spmm_args {
    int32_t n_rows, n_src;
    int32_t width;                     /* W >= 1 */
    int64_t nnz;                       /* < 2^31 */
    const int32_t *d_indptr;           /* [n_rows+1] */
    const int32_t *d_indices;          /* [nnz] in [0, n_src) */
    const float *d_values;             /* [nnz] */
    const int32_t *d_order;            /* [n_rows] a permutation of the rows */
    const float *d_dense;              /* D [n_src][W] */
    float *d_out;                      /* Y [n_rows][W], must not overlap D */
} lk_spmm_args;

LK_API int lk_spmm(const lk_spmm_args *args, void *stream);

/* ------------------------------------------------------------------------
 * NMF coordinate descent (nmf.cu), scikit-learn's solver="cd" behind NMFScorer (src/lenskit/sklearn/nmf.py).
 *
 * lk_nmf_cd_sweep is one `_update_cdnmf_fast(W, HHt, XHt, arange(k))` bit for bit: for each component t in
 * order and each row i,
 *     grad = -XHt[i][t];  for r in 0..k-1: grad = grad + HHt[t][r] * W[i][r]      (product and sum each rounded)
 *     pg = W[i][t] == 0 ? min(0, grad) : grad;   d_pg[t][i] = |pg|
 *     if HHt[t][t] != 0: W[i][t] = max(W[i][t] - grad / HHt[t][t], 0)
 * W is updated in place.  The sweep's violation is the left-to-right f32 sum of d_pg in its [k][n] order, which
 * lk_f32_seq_sum computes.  k in 1..128, else LK_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------- */
typedef struct lk_nmf_cd_sweep_args {
    int32_t n;                         /* rows of W */
    int32_t k;                         /* components, 1..128 */
    float *d_w;                        /* W [n][k] row-major, in place */
    const float *d_hht;                /* HHt [k][k] row-major, l2 already on the diagonal */
    const float *d_xht;                /* XHt [n][k] row-major, l1 already subtracted */
    float *d_pg;                       /* [k][n] out: |projected gradient|, component-major */
} lk_nmf_cd_sweep_args;

LK_API int lk_nmf_cd_sweep(const lk_nmf_cd_sweep_args *args, void *stream);

/* lk_f32_seq_sum: `count` (1..8) independent sums, run concurrently, one CTA each.  Sum i is
 *     s = +0.0f;  for j in 0..n-1: s = s + x[j]      (each addition rounded to nearest even)
 * over non-negative values (inf and NaN propagate as in that loop), which is np.cumsum(x, dtype=float32)[-1]
 * bit for bit, written to *d_out.  It needs no workspace: each sum is scanned one tile at a time within its CTA. */
typedef struct lk_f32_seq_sum_args {
    int64_t n;
    const float *d_x;                  /* [n] */
    float *d_out;                      /* [1] */
} lk_f32_seq_sum_args;

LK_API int lk_f32_seq_sum(const lk_f32_seq_sum_args *sums, int32_t count, void *stream);

/* ------------------------------------------------------------------------
 * Bias model and offset scoring (basic.cu), behind BiasScorer and PopScorer (src/lenskit/basic/bias.py,
 * popularity.py).
 *
 * lk_bias_learn is BiasModel.learn (bias.py:84-150) bit for bit, on ratings r in (user, item) COO order:
 *     g = f32(f64(+0.0f + pairwise(r)) / nnz)          np.mean of the f32 ratings (NumPy's pairwise order)
 *     c = r - g                                        f32, or f64(r) - g with centered_f64
 *   item pass:  cnt = d_item; s = 0.0; for each rating of the item by ascending user: cnt += 1.0; s += f64(c)
 *               ib[i] = cnt > 0 ? f32(s / cnt) : 0;  then c = c - ib[item]   (in c's type)
 *   user pass:  the same over each user's ratings in COO order, ub[u] = cnt > 0 ? f32(s / cnt) : 0
 * Every add is a rounded f64 add in that order (np.add.at); the counts too, unless d is an integer, when they are
 * exactly d + n.  A pass left out (d_item_bias or d_user_bias NULL) is skipped; without the item pass the user
 * pass sums r - g.  The mean is a parallel walk of the pairwise tree; each entity's sum is one warp, with entities
 * handed out in the caller's order (longest first keeps the longest chains from starting last).
 * ---------------------------------------------------------------------- */
typedef struct lk_bias_learn_args {
    int64_t nnz;                       /* 1 .. 2^31 - 1 */
    int32_t n_users, n_items;
    const float *d_ratings;            /* [nnz] COO order, sorted by (user, item) */
    const int32_t *d_items;            /* [nnz] COO item numbers */
    const int32_t *d_user_indptr;      /* [n_users + 1] offsets of each user's ratings in COO order */
    const int32_t *d_item_indptr;      /* [n_items + 1] offsets into d_item_ratings */
    const float *d_item_ratings;       /* [nnz] the ratings item-major, ascending user within an item */
    const int32_t *d_user_order;       /* [n_users] every user once: the order users are handed to warps */
    const int32_t *d_item_order;       /* [n_items] every item once */
    int32_t centered_f64;              /* 0: c in f32 (an f32 rating matrix), 1: c in f64 */
    double damping_user, damping_item; /* >= 0 */
    void *d_workspace;                 /* lk_bias_learn_workspace_bytes() bytes */
    float *d_mean;                     /* [1] out: g */
    float *d_item_bias;                /* [n_items] out, or NULL: no item pass */
    float *d_user_bias;                /* [n_users] out, or NULL: no user pass */
} lk_bias_learn_args;

LK_API int64_t lk_bias_learn_workspace_bytes(void);
LK_API int lk_bias_learn(const lk_bias_learn_args *args, void *stream);

/*
 * lk_offset_score_batch: s(q, i) = f32(f64(base[i]) + offset[q]) for every item i and query q (offset NULL: 0).
 * With the offset in f64 that is NumPy's `f32 scores += f64 user bias` (computed in f64, rounded once) and, for an
 * f32 offset, the f32 sum itself.  n == 0: score mode, d_scores [B][n_items] row-major.  n in 1..lk_topn_max():
 * rank mode, argtopn over every item in ascending order (topn_heap.cuh's output contract), the query's exclusions
 * (ascending within each query, in range) and NaN scores never offered.  One thread per query.
 */
typedef struct lk_offset_score_args {
    int32_t n_items, n_queries;
    const float *d_base;               /* [n_items] */
    const double *d_offset;            /* [n_queries] or NULL */
    int32_t n;
    float *d_scores;                   /* score mode */
    const int64_t *d_excl_indptr;      /* rank mode: [B + 1] or NULL */
    const int32_t *d_excl_items;
    int32_t *d_out_idx;                /* [B][n] */
    float *d_out_val;                  /* [B][n] */
    int32_t *d_out_cnt;                /* [B] */
} lk_offset_score_args;

LK_API int lk_offset_score_batch(const lk_offset_score_args *args, void *stream);

/* ------------------------------------------------------------------------
 * Stochastic top-n (stochastic.cu), behind StochasticTopNRanker (src/lenskit/stochastic/_ranker.py:89-156).
 *
 * Each of B rows holds n_items f32 scores at d_scores[q * row_stride + i * item_stride] (a contiguous [B][L]
 * matrix, or the transpose of an item-major [L][B] one, without a copy).  Position i of row q is valid when its score
 * is finite and i is not among the row's exclusions (ascending, in range; topn_excluded's semantics).  With N valid
 * positions, numbered in list order, and s = f32(score * scale):
 *   LK_STOCH_SOFTMAX  e = f32(exp(f64(s - max s)));  w = e / (+0.0f + pairwise(e))               (f32)
 *   LK_STOCH_LINEAR   r = f64(max s) - f64(min s); t = (s - min s) / f32(r); w = t / (+0.0f + pairwise(t));
 *                     w = 1.0f / f32(N) when !(r > 0) or !(sum > 0)                              (f32)
 *   LK_STOCH_NONE     w = s
 *   key = log(u) / f64(max(w, FLT_MIN))   (f64), u = (raw >> 11) * 2^-53 the k-th draw of the query's stream for
 *   the k-th valid position, raw = XSL-RR of the PCG64 state after the draw's step (NumPy's PCG64: the 128-bit LCG
 *   state = state * M + inc, then the output of the new state).  pairwise is NumPy's order (pairwise.cuh) over
 *   the valid values in list order.  A row with nothing valid draws nothing.
 * Streams: d_state holds (state_hi, state_lo, inc_hi, inc_lo).  shared_stream = 0: row q draws from its own state
 *   d_state[4q .. 4q+3] from its start.  shared_stream = 1: every row draws from d_state[0 .. 3], row q starting
 *   after the draws of rows 0 .. q-1 and *d_position draws in; *d_position is advanced by the batch's draws, so a
 *   batch split into calls continues one stream, and the caller reads the total from it once.
 * d_jump: lk_stochastic_jump_words() u64, built by the caller: entries 0..32 are (M^j, G_j) and entries 33..96 are
 *   (M^(2^t), G_(2^t)), each as (mul_hi, mul_lo, add_hi, add_lo), where G_j = sum_{k<j} M^k: j steps take s to
 *   M^j s + G_j inc (mod 2^128).
 * n in 1..lk_topn_max(): rank mode, argtopn over the keys with the valid positions offered in list order
 *   (topn_heap.cuh's contract): d_out_idx [B][n] positions (-1 padding), d_out_val [B][n] the original scores (NaN
 *   padding), d_out_key [B][n] the keys (NaN padding; may be NULL), d_out_cnt [B] the list lengths.
 * n == 0: key mode, d_keys [B][n_items] row-major, the key of every valid position and NaN elsewhere; d_out_cnt [B]
 *   the valid counts.
 * The workspace is lk_stochastic_workspace_bytes(B, n_items, transform) bytes: 20 per row, plus 4 * B * n_items for
 * the compacted values that softmax and linear sum.  Callers split large batches to bound it.
 * ---------------------------------------------------------------------- */
#define LK_STOCH_NONE 0
#define LK_STOCH_SOFTMAX 1
#define LK_STOCH_LINEAR 2
#define LK_STOCH_JUMP_WORDS (4 * (33 + 64))

typedef struct lk_stochastic_args {
    int32_t n_queries, n_items;        /* B rows of n_items positions (n_items < 2^31 - 64) */
    const float *d_scores;
    int64_t row_stride, item_stride;   /* in elements */
    const int64_t *d_excl_indptr;      /* [B + 1] or NULL */
    const int32_t *d_excl_items;
    int32_t transform;                 /* LK_STOCH_* */
    float scale;
    int32_t shared_stream;             /* 0: a state per row, 1: one stream through the rows */
    int32_t n;                         /* 0: key mode, 1..lk_topn_max(): rank mode */
    const uint64_t *d_state;           /* [B][4], or [1][4] with shared_stream */
    const uint64_t *d_jump;            /* [LK_STOCH_JUMP_WORDS] */
    int64_t *d_position;               /* shared_stream: [1] in/out, draws consumed */
    void *d_workspace;
    int64_t workspace_bytes;
    int32_t *d_out_idx;                /* rank mode [B][n] */
    float *d_out_val;                  /* rank mode [B][n] */
    double *d_out_key;                 /* rank mode [B][n], or NULL */
    int32_t *d_out_cnt;                /* [B] */
    double *d_keys;                    /* key mode [B][n_items] */
} lk_stochastic_args;

LK_API int64_t lk_stochastic_workspace_bytes(int64_t n_queries, int64_t n_items, int32_t transform);
LK_API int lk_stochastic_topn(const lk_stochastic_args *args, void *stream);

/* ------------------------------------------------------------------------
 * FA*IR re-ranking (fair.cu), behind FAIRReranker.__call__ (src/lenskit/reranking/fair.py).
 *
 * The merge of one ranked list of L positions with protected flags f[0 .. L) and a length len <= L: with P the
 * queue of protected positions and U the queue of the others, both ascending, and c the protected count so far,
 * for i = 0 .. len-1 take the head of P when c < d_m[i] and P is not empty, else the smaller head of P and U (the
 * head of whichever is not empty).  Scores are never read by the merge.
 *
 * mode LK_FAIR_LISTS: B lists, list b the positions d_list_indptr[b] .. d_list_indptr[b+1] of d_list_protected
 *   (one byte per position, nonzero = protected), merged to length d_list_len[b] (0 .. min(n, list length)).
 *   Output: d_out_idx [B][n] the chosen positions within each list, -1 padding; d_out_cnt [B] = d_list_len.
 * mode LK_FAIR_SCORES: B rows of n_items f32 scores at d_scores[q * row_stride + i * item_stride], one protected
 *   byte per item (d_item_protected [n_items]), optional exclusions (d_excl_indptr [B + 1] and d_excl_items,
 *   ascending and in range within each row, topn_excluded's semantics).  Each row's list is argtopn's top
 *   n_candidates (1 .. lk_topn_max()) of its scores, an excluded item offered as NaN (topn_heap.cuh's contract),
 *   and the merge runs over that list to length min(n, its length).  Output in argtopn's contract: d_out_idx [B][n]
 *   item numbers (-1 padding), d_out_val [B][n] their scores (NaN padding; may be NULL), d_out_cnt [B].
 * n in 1 .. lk_topn_max(); d_m holds at least n entries (the trained m_list).
 * ---------------------------------------------------------------------- */
#define LK_FAIR_LISTS 0
#define LK_FAIR_SCORES 1

typedef struct lk_fair_args {
    int32_t mode;                      /* LK_FAIR_* */
    int32_t n_queries;                 /* B */
    int32_t n;                         /* output width, 1..lk_topn_max() */
    int32_t n_candidates;              /* scores: N, 1..lk_topn_max() */
    const int32_t *d_m;                /* [n] minimum protected counts of the prefixes 1..n */
    const int64_t *d_list_indptr;      /* lists: [B + 1] */
    const uint8_t *d_list_protected;   /* lists: one flag per position */
    const int32_t *d_list_len;         /* lists: [B] output lengths */
    int32_t n_items;                   /* scores */
    const float *d_scores;             /* scores */
    int64_t row_stride, item_stride;   /* scores, in elements */
    const uint8_t *d_item_protected;   /* scores: [n_items] */
    const int64_t *d_excl_indptr;      /* scores: [B + 1] or NULL */
    const int32_t *d_excl_items;
    int32_t *d_out_idx;                /* [B][n] */
    float *d_out_val;                  /* scores: [B][n] or NULL */
    int32_t *d_out_cnt;                /* [B] */
} lk_fair_args;

LK_API int lk_fair_rerank(const lk_fair_args *args, void *stream);

/* ------------------------------------------------------------------------
 * Ranking metrics (metrics.cu), behind the measure_list of src/lenskit/metrics/ranking's metric classes.
 *
 * lk_rank_metrics: B lists, list b the item numbers d_rec_items[d_rec_indptr[b] .. d_rec_indptr[b+1]) in rank
 *   order (-1: an item the numbering does not know, never good), its test set d_test_items[d_test_indptr[b] ..
 *   d_test_indptr[b+1]) (known numbers, ascending, unique) and nrel = d_nrel[b], the test list's length as the
 *   reference counts it (unknown and repeated ids included).  Metric m truncates list b to k = min(L, n) positions
 *   (n = -1: k = L; every k at most lk_topn_max()), with g good positions among them at 0-based positions p_j:
 *     HIT          NaN if nrel = 0, else 1 if g > 0 else 0
 *     PRECISION    NaN if k = 0, else g / k
 *     RECALL       g / d, d = min(nrel, n) (n = -1: nrel); NaN if d = 0
 *     RECIP_RANK   NaN if nrel = 0, 0 if g = 0, else 1 / (p_0 + 1)
 *     DCG          NaN if nrel = 0, else S = pairwise_j(w[p_j])
 *     NDCG         S / norms[m], m = min(nrel, n) for n > 0, else nrel
 *     RBP          S / series_sum, S / norms[min(nrel, k)] (LK_RBP_NORM_PREFIX) or S / norms[k] (LK_RBP_NORM_LIST)
 *     AP           NaN if k = 0, else pairwise_j((j + 1) / (p_j + 1)) / min(nrel, k)
 *     MEAN_POP_RANK NaN if k = 0, else pairwise_{i < k}(w[item_i], 0 for item -1) / k
 *   with w = d_weights + weight_offset and norms = d_norms + norm_offset, which the caller sizes for every index
 *   read; pairwise is NumPy's order (pairwise.cuh) and every operation rounds to nearest.  Output d_out [M][B].
 * lk_item_exposure: the per-item totals of n_entries (item, rank) entries sorted stably by item (d_sorted_items
 *   ascending, d_order the sort's permutation of the entries, d_entry_list and d_entry_rank each entry's list and
 *   0-based rank, in entry order).  Of several entries of one item in one list only the last counts (NumPy's
 *   `totals[items] += values` with a repeated index).  d_totals[i] = the number of counted entries of item i when
 *   d_weights is NULL, else 0.0 + w[rank] of its counted entries added one by one in entry order.
 * ---------------------------------------------------------------------- */
#define LK_METRIC_HIT 0
#define LK_METRIC_PRECISION 1
#define LK_METRIC_RECALL 2
#define LK_METRIC_RECIP_RANK 3
#define LK_METRIC_DCG 4
#define LK_METRIC_NDCG 5
#define LK_METRIC_RBP 6
#define LK_METRIC_AP 7
#define LK_METRIC_MEAN_POP_RANK 8
#define LK_RBP_NORM_SERIES 0
#define LK_RBP_NORM_PREFIX 1
#define LK_RBP_NORM_LIST 2
#define LK_RANK_METRICS_MAX 32

typedef struct lk_metric_spec {
    int32_t kind;                      /* LK_METRIC_* */
    int32_t n;                         /* truncation, -1 for none */
    int64_t weight_offset;             /* into d_weights */
    int64_t norm_offset;               /* into d_norms */
    int32_t norm_mode;                 /* RBP: LK_RBP_NORM_* */
    int32_t reserved;
    double series_sum;                 /* RBP with LK_RBP_NORM_SERIES */
} lk_metric_spec;

typedef struct lk_rank_metrics_args {
    int64_t n_lists;                   /* B */
    const int64_t *d_rec_indptr;       /* [B + 1] */
    const int32_t *d_rec_items;
    const int64_t *d_test_indptr;      /* [B + 1] */
    const int32_t *d_test_items;
    const int64_t *d_nrel;             /* [B] */
    const double *d_weights;
    const double *d_norms;
    double *d_out;                     /* [M][B] */
    int32_t n_metrics;                 /* M, 0..LK_RANK_METRICS_MAX */
    int32_t reserved;
    lk_metric_spec metrics[LK_RANK_METRICS_MAX];
} lk_rank_metrics_args;

typedef struct lk_item_exposure_args {
    int64_t n_items;
    int64_t n_entries;
    const int32_t *d_sorted_items;     /* [n_entries] ascending */
    const int64_t *d_order;            /* [n_entries] */
    const int32_t *d_entry_list;       /* [n_entries], in entry order */
    const int32_t *d_entry_rank;       /* [n_entries], in entry order */
    const double *d_weights;           /* by rank, or NULL */
    double *d_totals;                  /* [n_items] */
} lk_item_exposure_args;

LK_API int lk_rank_metrics(const lk_rank_metrics_args *args, void *stream);
LK_API int lk_item_exposure(const lk_item_exposure_args *args, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* LKPY_B200_H */
