// cooc.cu — co-occurrence counting and association scoring for sm_90a.
//
// Counting replaces count_cooc_parallel (src/accel/data/cooc.rs:185-214), which walks the groups serially and
// makes one atomic increment per position pair into an n(n+1)/2 int32 triangle.  Here the shared tile core
// (tiles.cuh) builds row i from i's group occurrences (IG) as the input rows and, for each, the group's items (GI)
// inside the warp's column sub-tile, found through lk_knn_tile_pointers.  A warp owns a contiguous sub-tile of
// uint32 counters in shared memory; integer addition commutes, so the lanes add with shared-memory atomics in any
// order.  Keeping repeated items in both GI and IG makes the reference's duplicate
// semantics (sum_g #i * #j off the diagonal) fall out of the enumeration.  Work units are (item, column tile),
// handed out most-expensive-first by a persistent grid; the strict upper triangle skips the tiles left of the
// diagonal.  After a unit the warps compact their non-zero counters (ballot + popcount keep column order) into
// one bump-allocated pool segment, optionally turned into the association value (the f64-divide chain of
// association.py:117-124) on the way, and lk_cooc_pool_to_csr gathers the segments into a row-sorted CSR.
//
// Scoring replaces AssociationScorer.__call__ (and, as a plain sum, SLIMScorer.__call__'s x @ weights): one CTA per
// (query, column tile) in score mode, one CTA per
// query sweeping the column tiles in ascending order in rank mode.  Each warp owns a sub-tile of f32
// accumulators and walks the query's reference rows in query order (the input rows of the tile core, applied one
// row per round), so every accumulator sees the same sequence of f32
// adds as NumPy's np.mean(axis=0) over the dense rows (absent entries add +0.0, which changes nothing).  In rank
// mode warp 0 then offers the tile's scores in ascending item order to argtopn's heap (topn_heap.cuh), keeping
// only count < n || s > root (exact: a full heap's root never decreases and a full heap rejects s <= root) and
// skipping NaN scores (+inf and -inf in two reference rows at one column) and excluded items (argtopn's NaN offer).
#include "tiles.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int CO_WARPS = 16;
constexpr int CO_NT = CO_WARPS * 32;
constexpr int CO_CTAS = 2;

constexpr int CO_FIXED_SMEM = TOPN_MAX * 8 + CO_WARPS * 4 + 16;  // argtopn heap, per-warp counts

static int co_smem_bytes(const lk_knn_geom &g) { return g.warps * g.tile_cols * 4 + CO_FIXED_SMEM; }

__global__ void cooc_row_cost_kernel(const lk_cooc_args a, int64_t *__restrict__ cost)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.geom.n_items; i += warps) {
        long long s = 0;
        for (int p = a.d_ig_indptr[i] + lane; p < a.d_ig_indptr[i + 1]; p += 32) {
            const int g = a.d_ig_groups[p];
            const int lo0 = a.d_gi_indptr[g], hi = a.d_gi_indptr[g + 1];
            int lo = lo0;
            if (!a.full_rows) {  // first column > i
                int h2 = hi;
                while (lo < h2) {
                    const int mid = (lo + h2) >> 1;
                    if (a.d_gi_items[mid] <= i) lo = mid + 1; else h2 = mid;
                }
            }
            s += hi - lo;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
        if (lane == 0) cost[i] = s;
    }
}

__device__ __forceinline__ uint32_t assoc_bits(uint32_t count, double row_den, const lk_cooc_args &a, int c,
                                               float n_groups)
{
    float v = __double2float_rn(__ddiv_rn((double)__uint2float_rn(count), row_den));
    if (a.method == LK_ASSOC_LIFT) {
        v = __fmul_rn(v, n_groups);
        v = __double2float_rn(__ddiv_rn((double)v, __dadd_rn((double)a.d_item_count[c], a.damping)));
    }
    return __float_as_uint(v);
}

__global__ void __launch_bounds__(CO_NT, CO_CTAS) cooc_count_kernel(const lk_cooc_args a)
{
    constexpr int W = CO_WARPS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ int s_work;
    const lk_knn_geom &g = a.geom;
    const int TW = g.tile_cols, S1 = g.n_subtiles + 1, H = g.n_halves;
    uint32_t *acc = reinterpret_cast<uint32_t *>(smem_raw);  // [W * TW]
    int *wcnt = reinterpret_cast<int *>(acc + W * TW);         // [W]
    const float n_groups = (float)g.n_users;  // NumPy's f32 array * Python int

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int idx = tid; idx < W * TW; idx += CO_NT) acc[idx] = 0u;
    __syncthreads();

    for (;;) {
        const int64_t wi = cta_next_work(a.d_work_counter, a.d_cancel, &s_work);
        if (wi >= a.n_work) break;
        const int unit = a.d_sched[wi];
        const int item = unit / H, h = unit - item * H;
        const int s = h * W + warp;  // this warp's sub-tile: columns [col0, col0 + TW)
        const int col0 = s * TW;
        uint32_t *my = acc + warp * TW;
        const int lo_col = a.full_rows ? 0 : item + 1;  // columns below lo_col are not counted

        bool any = false;
        if (col0 + TW > lo_col) {
            const int p0 = a.d_ig_indptr[item];
            const int m = a.d_ig_indptr[item + 1] - p0;
            for (int t0 = 0; t0 < m; t0 += 32) {
                int len = 0, base = 0;
                if (t0 + lane < m) {
                    const int grp = __ldg(a.d_ig_groups + p0 + t0 + lane);
                    const int32_t *tp = a.d_tile_ptr + (size_t)grp * S1 + s;
                    base = __ldg(tp);
                    len = __ldg(tp + 1) - base;
                }
                any |= warp_walk_segments(base, len, lane, [&](bool valid, int, int src) {
                    if (valid) {
                        const int col = __ldg(a.d_gi_items + src);
                        if (col >= lo_col && col != item) atomicAdd(&my[col - col0], 1u);
                    }
                });
            }
        }
        if (!__syncthreads_or(any)) {  // no group of the item reaches this tile: every counter is still 0
            if (tid == 0) {
                a.d_part_cnt[unit] = 0;
                a.d_pool_off[unit] = 0;
            }
            continue;
        }

        const double row_den = a.method != LK_COOC_COUNT ? __dadd_rn((double)a.d_item_count[item], a.damping) : 1.0;
        cta_emit_pool_segment<W>(
            my, TW, col0, unit, [](uint32_t v, int) { return v != 0u; },
            [&](uint32_t v, int c) { return a.method == LK_COOC_COUNT ? v : assoc_bits(v, row_den, a, c, n_groups); },
            0u, wcnt, a.d_pool_cursor, a.pool_capacity, a.d_status, a.d_pool_off, a.d_part_cnt, a.d_pool_cols,
            static_cast<uint32_t *>(a.d_pool_vals));
    }
}

// one thread per group: runs of an item inside the group's ascending list give #i (#i + 1) / 2
__global__ void cooc_diag_kernel(const lk_cooc_args a, unsigned long long *__restrict__ diag)
{
    const int stride = gridDim.x * blockDim.x;
    for (int grp = blockIdx.x * blockDim.x + threadIdx.x; grp < a.geom.n_users; grp += stride) {
        const int hi = a.d_gi_indptr[grp + 1];
        int p = a.d_gi_indptr[grp];
        while (p < hi) {
            const int it = a.d_gi_items[p];
            int q = p + 1;
            while (q < hi && a.d_gi_items[q] == it) q++;
            const unsigned long long c = (unsigned long long)(q - p);
            atomicAdd(diag + it, c * (c + 1) / 2);
            p = q;
        }
    }
}

__global__ void cooc_dense_kernel(int n, const int64_t *__restrict__ indptr, const int32_t *__restrict__ cols,
                                  const int32_t *__restrict__ counts, const int64_t *__restrict__ diag,
                                  float *__restrict__ out)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        for (int64_t p = indptr[i] + lane; p < indptr[i + 1]; p += 32) {
            const int64_t j = cols[p];
            const float v = (float)counts[p];
            out[(int64_t)i * n + j] = v;
            out[j * n + i] = v;
        }
        if (diag != nullptr && lane == 0) out[(int64_t)i * n + i] = (float)diag[i];
    }
}

__global__ void assoc_tile_ptr_kernel(const lk_knn_geom g, const int64_t *__restrict__ indptr,
                                      const int32_t *__restrict__ cols, int32_t *__restrict__ tptr)
{
    const int64_t S1 = g.n_subtiles + 1;
    const int64_t total = (int64_t)g.n_users * S1;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(idx / S1), s = (int)(idx % S1);
        const int64_t bound = (int64_t)s * g.tile_cols, r0 = indptr[r];
        int64_t lo = r0, hi = indptr[r + 1];
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)cols[mid] < bound) lo = mid + 1; else hi = mid;
        }
        tptr[idx] = (int32_t)(lo - r0);  // a row has fewer than 2^31 columns
    }
}

template <bool RANK>
__global__ void __launch_bounds__(CO_NT, CO_CTAS) assoc_score_kernel(const lk_assoc_score_args a)
{
    constexpr int W = CO_WARPS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const lk_knn_geom &g = a.geom;
    const int TW = g.tile_cols, S1 = g.n_subtiles + 1, H = g.n_halves, NI = g.n_items;
    const int CW = W * TW;
    float *acc = reinterpret_cast<float *>(smem_raw);  // [CW]
    PairHeap<1> heap{acc + CW, reinterpret_cast<int32_t *>(acc + CW + TOPN_MAX)};

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q = RANK ? (int)blockIdx.x : (int)(blockIdx.x / H);
    const int h_first = RANK ? 0 : (int)(blockIdx.x % H), h_end = RANK ? H : h_first + 1;
    const int64_t r0 = a.d_ref_indptr[q];
    const int R = (int)(a.d_ref_indptr[q + 1] - r0);
    const float qnan = __int_as_float(0x7fc00000);
    const int n = a.n;

    if (R == 0 && a.agg != 2) {  // no reference items: every score is NaN, nothing is recommended (a sum is +0.0)
        if constexpr (RANK) {
            for (int t = tid; t < n; t += CO_NT) {
                a.d_out_idx[(int64_t)q * n + t] = -1;
                a.d_out_val[(int64_t)q * n + t] = qnan;
            }
            if (tid == 0) a.d_out_cnt[q] = 0;
        } else {
            for (int j = tid; j < CW; j += CO_NT) {
                const int c = h_first * CW + j;
                if (c < NI) a.d_scores[(int64_t)q * NI + c] = qnan;
            }
        }
        return;
    }

    for (int j = tid; j < CW; j += CO_NT) acc[j] = 0.0f;
    __syncthreads();

    int count = 0;  // rank mode, warp 0: heap size and root, exclusion cursor
    float root = 0.0f;
    int64_t ec = 0, ee = 0;
    if (RANK && a.d_excl_indptr != nullptr) ec = a.d_excl_indptr[q], ee = a.d_excl_indptr[q + 1];

    for (int h = h_first; h < h_end; h++) {
        const int s = h * W + warp;
        const int col0 = s * TW;
        float *my = acc + warp * TW;
        for (int t0 = 0; t0 < R; t0 += 32) {
            int len = 0;
            int64_t base = 0;
            if (t0 + lane < R) {
                const int r = __ldg(a.d_ref_items + r0 + t0 + lane);
                const int32_t *tp = a.d_tile_ptr + (size_t)r * S1 + s;
                const int b0 = __ldg(tp);
                base = __ldg(a.d_indptr + r) + b0;
                len = __ldg(tp + 1) - b0;
            }
            warp_walk_segments(base, len, lane, [&](bool valid, int own, int64_t src) {
                int j = 0;
                float v = 0.0f;
                if (valid) {
                    j = __ldg(a.d_cols + src) - col0;
                    v = __ldg(a.d_vals + src);
                }
                // reference rows in query order
                warp_apply_in_owner_order(valid, own, [&] {
                    my[j] = a.agg != 1 ? __fadd_rn(my[j], v) : fmaxf(my[j], v);
                });
            });
        }
        // final scores of the warp's sub-tile: np.mean divides the f32 sum by the row count in f64
        if (a.agg == 0) {
            for (int c0 = lane; c0 < TW; c0 += 32)
                my[c0] = __double2float_rn(__ddiv_rn((double)my[c0], (double)R));
        }
        __syncwarp();
        if constexpr (!RANK) {
            for (int c0 = lane; c0 < TW; c0 += 32) {
                const int c = col0 + c0;
                if (c < NI) a.d_scores[(int64_t)q * NI + c] = my[c0];
                my[c0] = 0.0f;
            }
        } else {
            __syncthreads();
            if (warp == 0) {
                const int32_t *ex = a.d_excl_items;
                for (int j0 = 0; j0 < CW; j0 += 32) {
                    const int c = h * CW + j0 + lane;
                    const float sc = acc[j0 + lane];
                    unsigned b = __ballot_sync(FULL, c < NI && sc == sc && (count < n || sc > root));
                    if (lane == 0) {
                        while (b) {
                            const int l = __ffs(b) - 1;
                            b &= b - 1u;
                            const int item = h * CW + j0 + l;
                            if (topn_excluded(ex, ec, ee, item)) continue;  // argtopn's NaN offer
                            topn_heap_offer(heap, count, root, n, PairHeap<1>::Ent{acc[j0 + l], item});
                        }
                    }
                    count = __shfl_sync(FULL, count, 0);
                    root = __shfl_sync(FULL, root, 0);
                }
            }
            __syncthreads();
            for (int j = tid; j < CW; j += CO_NT) acc[j] = 0.0f;
            __syncthreads();
        }
    }

    if constexpr (RANK) {
        if (tid == 0) {
            topn_heap_sort(heap, count);
            const int64_t o = (int64_t)q * n;
            for (int t = 0; t < n; t++) {
                const bool in = t < count;
                a.d_out_idx[o + t] = in ? heap.hk[t] : -1;
                a.d_out_val[o + t] = in ? heap.hv[t] : qnan;
            }
            a.d_out_cnt[q] = count;
        }
    }
}

template <bool RANK>
int launch_assoc_score(const lk_assoc_score_args &a, cudaStream_t st)
{
    const int smem = co_smem_bytes(a.geom);
    LK_CUDA_TRY(cudaFuncSetAttribute(assoc_score_kernel<RANK>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const unsigned grid = RANK ? (unsigned)a.n_queries : (unsigned)((int64_t)a.n_queries * a.geom.n_halves);
    assoc_score_kernel<RANK><<<grid, CO_NT, smem, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_cooc_geometry(int32_t n_rows, int32_t n_cols, lk_knn_geom *geom)
{
    LK_REQUIRE(geom != nullptr && n_rows >= 0 && n_cols >= 1, LK_ERR_INVALID, "lk_cooc_geometry: bad arguments");
    // 4-byte accumulators; the argtopn heap of the scoring kernel's rank mode is reserved in every geometry
    tile_geometry(n_rows, n_cols, CO_WARPS, CO_CTAS, 4, CO_FIXED_SMEM, 64, geom);
    return LK_OK;
}

static int cooc_check(const lk_cooc_args *args, const char *who)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "%s: null args", who);
    const lk_cooc_args &a = *args;
    LK_REQUIRE(a.geom.warps == CO_WARPS && a.geom.n_halves >= 1, LK_ERR_INVALID, "%s: geometry not from lk_cooc_geometry",
               who);
    LK_REQUIRE((int64_t)a.geom.n_items * a.geom.n_halves < 0x7fffffffLL, LK_ERR_UNSUPPORTED,
               "%s: n_items * n_halves must be < 2^31", who);
    LK_REQUIRE(a.d_gi_indptr && a.d_gi_items && a.d_ig_indptr && a.d_ig_groups, LK_ERR_INVALID, "%s: null matrix", who);
    return LK_OK;
}

int lk_cooc_row_cost(const lk_cooc_args *args, int64_t *d_cost, void *stream)
{
    if (int rc = cooc_check(args, "lk_cooc_row_cost")) return rc;
    LK_REQUIRE(d_cost != nullptr, LK_ERR_INVALID, "lk_cooc_row_cost: null cost");
    cooc_row_cost_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, d_cost);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_cooc_count(const lk_cooc_args *args, void *stream)
{
    if (int rc = cooc_check(args, "lk_cooc_count")) return rc;
    const lk_cooc_args &a = *args;
    LK_REQUIRE(a.d_work_counter && a.d_status && a.d_pool_cursor, LK_ERR_INVALID, "lk_cooc_count: null counter");
    LK_REQUIRE(a.method == LK_COOC_COUNT || a.method == LK_ASSOC_PROBABILITY || a.method == LK_ASSOC_LIFT,
               LK_ERR_INVALID, "lk_cooc_count: unknown method %d", a.method);
    if (a.method != LK_COOC_COUNT) {
        LK_REQUIRE(a.full_rows && a.d_item_count != nullptr, LK_ERR_INVALID,
                   "lk_cooc_count: association values need full rows and the item counts");
        LK_REQUIRE(a.damping >= 0.0, LK_ERR_INVALID, "lk_cooc_count: damping must be non-negative");
    }
    LK_REQUIRE(a.max_row_cost >= 0 && a.max_row_cost < 0x80000000LL, LK_ERR_UNSUPPORTED,
               "lk_cooc_count: a row makes %lld pair updates; counts must stay below 2^31", (long long)a.max_row_cost);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_status, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
    if (a.n_work == 0) return LK_OK;
    LK_REQUIRE(a.d_tile_ptr && a.d_sched && a.d_pool_cols && a.d_pool_vals && a.d_pool_off && a.d_part_cnt,
               LK_ERR_INVALID, "lk_cooc_count: null pointer");
    const int smem = co_smem_bytes(a.geom);
    int64_t grid = (int64_t)sm_count() * CO_CTAS;
    if (grid > a.n_work) grid = a.n_work;
    LK_CUDA_TRY(cudaFuncSetAttribute(cooc_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cooc_count_kernel<<<(unsigned)grid, CO_NT, smem, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_cooc_pool_to_csr(const lk_cooc_args *args, const int64_t *d_out_indptr, int32_t *d_out_cols, void *d_out_vals,
                        void *stream)
{
    if (int rc = cooc_check(args, "lk_cooc_pool_to_csr")) return rc;
    LK_REQUIRE(d_out_indptr && d_out_cols && d_out_vals && args->d_pool_off && args->d_part_cnt, LK_ERR_INVALID,
               "lk_cooc_pool_to_csr: null pointer");
    const lk_cooc_args &a = *args;
    return launch_pool_to_csr(a.geom.n_items, a.geom.n_halves, a.d_pool_off, a.d_part_cnt, a.d_pool_cols,
                              static_cast<const uint32_t *>(a.d_pool_vals), d_out_indptr, d_out_cols,
                              static_cast<uint32_t *>(d_out_vals), stream);
}

int lk_cooc_diagonal(const lk_cooc_args *args, int64_t *d_diag, void *stream)
{
    if (int rc = cooc_check(args, "lk_cooc_diagonal")) return rc;
    LK_REQUIRE(d_diag != nullptr, LK_ERR_INVALID, "lk_cooc_diagonal: null output");
    if (args->geom.n_users == 0) return LK_OK;
    cooc_diag_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        *args, reinterpret_cast<unsigned long long *>(d_diag));
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_cooc_dense(int32_t n_items, const int64_t *d_indptr, const int32_t *d_cols, const int32_t *d_counts,
                  const int64_t *d_diag, float *d_out, void *stream)
{
    LK_REQUIRE(n_items >= 0 && d_indptr && d_cols && d_counts && d_out, LK_ERR_INVALID, "lk_cooc_dense: bad arguments");
    if (n_items == 0) return LK_OK;
    cooc_dense_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(n_items, d_indptr, d_cols,
                                                                                   d_counts, d_diag, d_out);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_assoc_tile_pointers(const lk_knn_geom *geom, const int64_t *d_indptr, const int32_t *d_cols,
                           int32_t *d_tile_ptr, void *stream)
{
    LK_REQUIRE(geom && d_indptr && d_tile_ptr, LK_ERR_INVALID, "lk_assoc_tile_pointers: null");
    if (geom->n_users == 0) return LK_OK;
    assoc_tile_ptr_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*geom, d_indptr, d_cols,
                                                                                       d_tile_ptr);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_assoc_score_batch(const lk_assoc_score_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_assoc_score_batch: null args");
    const lk_assoc_score_args &a = *args;
    LK_REQUIRE(a.geom.warps == CO_WARPS && a.geom.n_halves >= 1 && a.geom.n_users == a.geom.n_items, LK_ERR_INVALID,
               "lk_assoc_score_batch: geometry not from lk_cooc_geometry(n_items, n_items)");
    LK_REQUIRE(a.agg >= 0 && a.agg <= 2, LK_ERR_INVALID,
               "lk_assoc_score_batch: agg must be 0 (mean), 1 (max) or 2 (sum)");
    LK_REQUIRE(a.n_queries >= 0 && (int64_t)a.n_queries * a.geom.n_halves < 0x7fffffffLL, LK_ERR_UNSUPPORTED,
               "lk_assoc_score_batch: n_queries * n_halves must be < 2^31");
    const bool rank = a.n != 0;
    if (rank)
        LK_REQUIRE(a.n >= 1 && a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED,
                   "lk_assoc_score_batch: n must be 0 (score mode) or in 1..%d", TOPN_MAX);
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_indptr && a.d_cols && a.d_vals && a.d_tile_ptr && a.d_ref_indptr && a.d_ref_items, LK_ERR_INVALID,
               "lk_assoc_score_batch: null input");
    if (rank) {
        LK_REQUIRE(a.d_out_idx && a.d_out_val && a.d_out_cnt, LK_ERR_INVALID, "lk_assoc_score_batch: null output");
        LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
                   "lk_assoc_score_batch: d_excl_items is required with d_excl_indptr");
    } else {
        LK_REQUIRE(a.d_scores != nullptr, LK_ERR_INVALID, "lk_assoc_score_batch: null score matrix");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return rank ? launch_assoc_score<true>(a, st) : launch_assoc_score<false>(a, st);
}

}  // extern "C"
