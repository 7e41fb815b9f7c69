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
 *   _accel.data.argtopn (SURVEY.md 8f, "next")    src/accel/data/sorting.rs:131-170 lk_topn_columns
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
 * LK_ALS_TF32, LK_KNN_WARPS, LK_KNN_CTAS, LK_KNN_SCORE_SEQ, LK_KNN_SCORE_CTAS (meaning: lkpy_b200/csrc/common.cuh, struct Options). */
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
 * one warp nor unbalance the grid; chunks are ordered longest-row-first.  Each
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
    unsigned long long *d_prof; /* reserved (ignored by the kernels), NULL */
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
    float *d_acc_ws, *d_acc_tw;  /* [n_targets] accumulator scratch */
    int32_t *d_acc_cnt;          /* [n_targets] */
    float *d_scores;             /* [n_targets] NaN = null (Arrow null in the reference) */
    int32_t *d_counts;           /* [n_targets] -1 = null */
    int32_t *d_work_counter;     /* [1] zeroed by the call */
    int32_t *d_status;           /* [1] 0 ok; 2 NaN similarity */
    /* Per-warp heap states for the targets that receive more than max_nbrs contributions
     * (accum.rs:100-117): [slotmap_warps * heap_floats_per_warp] 32-bit words, 8-byte aligned;
     * one target takes 2 + 2*(max_nbrs+1) words.  Optional (NULL / 0): targets that do not fit are
     * replayed one at a time from the query's history instead (same result, much slower for long
     * histories). */
    float *d_heap_scratch;
    int64_t heap_floats_per_warp;
    /* Contribution pool (optional; with it the list-based kernel runs: per-target contribution
     * lists built in parallel, sorted by history position, replayed — same bits, no sequential
     * walk over the history).  pool_entries 16-byte entries, at least the number of
     * (reference item, similarity-row entry) pairs of the whole batch:
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
     * items in index order; d_scores / d_counts are [n_queries * n_items] and written exactly once, d_acc_cnt
     * is not used, the contribution pool is required.  A CTA handles a query and keeps its state per CTA:
     * d_slotmap provides one n_items row per CTA (slotmap_warps >= lk_knn_score_dense_ctas()) that must be
     * all ZERO on entry and is left all zero (item -> touched-target number), d_acc_ws / d_acc_tw one
     * n_items row per CTA each ([min(n_queries, lk_knn_score_dense_ctas()) * n_items] 32-bit words:
     * list offsets / cursors by touched-target number). */
    int32_t *d_deferred;         /* dense mode, optional: [n_queries] order in which the queries are handed to the CTAs
                                  * (a permutation; longest histories first keeps the tail of the launch short) */
    int32_t *d_n_deferred;       /* reserved (unused) */
} lk_knn_score_args;

/* largest number of warps the scoring grid runs (one slotmap row each) */
LK_API int64_t lk_knn_score_warps(void);
/* number of CTAs of the dense (all-items) scoring grid: one n_items row of d_slotmap each */
LK_API int64_t lk_knn_score_dense_ctas(void);
LK_API int lk_knn_score_batch(const lk_knn_score_args *args, void *stream);

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

#ifdef __cplusplus
}
#endif
#endif /* LKPY_B200_H */
