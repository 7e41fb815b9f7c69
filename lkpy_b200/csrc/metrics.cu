// metrics.cu — the ranking metrics of src/lenskit/metrics/ranking for batches of top-N lists (lk_rank_metrics), and
// the per-item totals that ListGini and ExposureGini accumulate (lk_item_exposure).
//
// lk_rank_metrics: one warp per list.  The warp tests each examined position against the list's test set (sorted
// and unique: a binary search per lane), and compacts the good positions, ascending, into shared memory with one
// ballot per 32 positions.  A truncation to k positions keeps a prefix of that array, so one pass serves every
// metric.  Then lane m computes metric m (at most LK_RANK_METRICS_MAX = 32 of them, their records passed by value)
// on its own: counts, the first good position, and sums in NumPy's pairwise order (pairwise.cuh) over the good
// positions in rank order, of entries of tables the host took from the reference's own weight classes.  Every add
// and division is an explicit round-to-nearest intrinsic.
//
// lk_item_exposure: one thread per item, over the entries the caller sorted stably by item (so each item's entries
// stay in list order): the item's total is 0.0 plus its weights added one by one, which is what the reference's
// repeated `totals[items] += weights` computes for it.  A count adds 1.0 the same way, which is exact.
#include "common.cuh"
#include "pairwise.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int METRIC_WARPS = 8;  // lists per CTA

__device__ __forceinline__ double metric_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

// is `item` in the sorted, unique set s[0 .. n)?
__device__ __forceinline__ bool sorted_member(const int32_t *s, const int64_t n, const int32_t item)
{
    if (item < 0) return false;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(s + mid) < item)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < n && __ldg(s + lo) == item;
}

// the number of entries of the ascending array a[0 .. n) below x
__device__ __forceinline__ int count_below(const int32_t *a, const int n, const int x)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < x)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// one metric of one list: L the list's length, good[0 .. G) its good positions (ascending) among the first
// min(L, TOPN_MAX) positions, nrel its test-set length as the reference counts it
__device__ double rank_metric(const lk_metric_spec &s, const lk_rank_metrics_args &a, const int32_t *recs,
                              const int L, const int32_t *good, const int G, const int64_t nrel)
{
    const int k = s.n < 0 ? L : min(L, s.n);
    const int g = count_below(good, G, k);  // good positions within the truncation
    const double *w = a.d_weights + s.weight_offset;
    const double *nm = a.d_norms + s.norm_offset;
    switch (s.kind) {
    case LK_METRIC_HIT:
        if (nrel == 0) return metric_nan();
        return g > 0 ? 1.0 : 0.0;
    case LK_METRIC_PRECISION:
        if (k == 0) return metric_nan();
        return __ddiv_rn((double)g, (double)k);
    case LK_METRIC_RECALL: {
        const int64_t d = (s.n >= 0 && s.n < nrel) ? s.n : nrel;
        if (d == 0) return metric_nan();  // 0 / 0
        return __ddiv_rn((double)g, (double)d);
    }
    case LK_METRIC_RECIP_RANK:
        if (nrel == 0) return metric_nan();
        if (g == 0) return 0.0;
        return __ddiv_rn(1.0, __dadd_rn((double)good[0], 1.0));
    case LK_METRIC_DCG:
    case LK_METRIC_NDCG:
    case LK_METRIC_RBP: {
        if (nrel == 0) return metric_nan();
        const double sum = pairwise_sum<F64Ops>([&](const int64_t j) { return __ldg(w + good[j]); }, 0, g);
        if (s.kind == LK_METRIC_DCG) return sum;
        if (s.kind == LK_METRIC_NDCG) {
            // fixed_dcg(m), m = min(nrel, n) for a positive n, else nrel
            const int64_t m = (s.n > 0 && s.n < nrel) ? s.n : nrel;
            return __ddiv_rn(sum, __ldg(nm + m));
        }
        if (s.norm_mode == LK_RBP_NORM_SERIES) return __ddiv_rn(sum, s.series_sum);
        const int64_t m = s.norm_mode == LK_RBP_NORM_PREFIX ? min((int64_t)k, nrel) : (int64_t)k;
        return __ddiv_rn(sum, __ldg(nm + m));
    }
    case LK_METRIC_AP: {
        if (k == 0) return metric_nan();
        // the running good count over the rank at each good position, summed in rank order
        const double sum = pairwise_sum<F64Ops>(
            [&](const int64_t j) { return __ddiv_rn((double)(j + 1), (double)(good[j] + 1)); }, 0, g);
        return __ddiv_rn(sum, (double)min((int64_t)k, nrel));
    }
    case LK_METRIC_MEAN_POP_RANK: {
        if (k == 0) return metric_nan();
        // the popularity quantile of each item in list order, 0 for an item outside the table
        const double sum = pairwise_sum<F64Ops>(
            [&](const int64_t j) {
                const int32_t it = __ldg(recs + j);
                return it >= 0 ? __ldg(w + it) : 0.0;
            },
            0, k);
        return __ddiv_rn(sum, (double)k);
    }
    default:
        return metric_nan();
    }
}

__global__ void __launch_bounds__(METRIC_WARPS * 32) rank_metrics_kernel(const lk_rank_metrics_args a)
{
    __shared__ int32_t good_smem[METRIC_WARPS][TOPN_MAX];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t b = (int64_t)blockIdx.x * METRIC_WARPS + wid;
    if (b >= a.n_lists) return;  // warp-uniform; the kernel has no barrier
    int32_t *good = good_smem[wid];

    const int64_t ro = __ldg(a.d_rec_indptr + b);
    const int L = (int)(__ldg(a.d_rec_indptr + b + 1) - ro);
    const int32_t *recs = a.d_rec_items + ro;
    const int64_t to = __ldg(a.d_test_indptr + b);
    const int64_t tn = __ldg(a.d_test_indptr + b + 1) - to;
    const int32_t *test = a.d_test_items + to;
    const int64_t nrel = __ldg(a.d_nrel + b);

    // the positions any metric reads: up to the longest truncation, at most TOPN_MAX (the host checks that)
    int scan = 0;
    for (int m = 0; m < a.n_metrics; m++) {
        const int n = a.metrics[m].n;
        scan = max(scan, n < 0 ? L : min(L, n));
    }
    scan = min(scan, TOPN_MAX);

    int G = 0;
    for (int base = 0; base < scan; base += 32) {
        const int p = base + lane;
        const bool hit = p < scan && sorted_member(test, tn, __ldg(recs + p));
        const unsigned mask = __ballot_sync(FULL, hit);
        if (hit) good[G + __popc(mask & ((1u << lane) - 1u))] = p;
        G += __popc(mask);
    }
    __syncwarp();

    for (int m = lane; m < a.n_metrics; m += 32)
        a.d_out[(int64_t)m * a.n_lists + b] = rank_metric(a.metrics[m], a, recs, L, good, G, nrel);
}

__global__ void item_exposure_kernel(const lk_item_exposure_args a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_items) return;
    // the item's run [lo, hi) of the sorted entries
    int64_t lo = 0, hi = a.n_entries;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(a.d_sorted_items + mid) < i)
            lo = mid + 1;
        else
            hi = mid;
    }
    int64_t end = lo, top = a.n_entries;
    while (end < top) {
        const int64_t mid = (end + top) >> 1;
        if (__ldg(a.d_sorted_items + mid) <= i)
            end = mid + 1;
        else
            top = mid;
    }
    // of an item's entries in one list (adjacent: the sort is stable) only the last counts
    double total = 0.0;
    for (int64_t j = lo; j < end; j++) {
        const int64_t e = __ldg(a.d_order + j);
        if (j + 1 < end && __ldg(a.d_entry_list + __ldg(a.d_order + j + 1)) == __ldg(a.d_entry_list + e)) continue;
        total = __dadd_rn(total, a.d_weights == nullptr ? 1.0 : __ldg(a.d_weights + __ldg(a.d_entry_rank + e)));
    }
    a.d_totals[i] = total;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_rank_metrics(const lk_rank_metrics_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_rank_metrics: null args");
    const lk_rank_metrics_args &a = *args;
    LK_REQUIRE(a.n_lists >= 0, LK_ERR_INVALID, "lk_rank_metrics: negative batch");
    LK_REQUIRE(a.n_metrics >= 0 && a.n_metrics <= LK_RANK_METRICS_MAX, LK_ERR_INVALID,
               "lk_rank_metrics: n_metrics must be in 0..%d", LK_RANK_METRICS_MAX);
    for (int m = 0; m < a.n_metrics; m++) {
        const lk_metric_spec &s = a.metrics[m];
        LK_REQUIRE(s.kind >= LK_METRIC_HIT && s.kind <= LK_METRIC_MEAN_POP_RANK, LK_ERR_INVALID,
                   "lk_rank_metrics: metric %d has unknown kind %d", m, s.kind);
        LK_REQUIRE(s.n >= -1, LK_ERR_INVALID, "lk_rank_metrics: metric %d has truncation %d", m, s.n);
        LK_REQUIRE(s.kind != LK_METRIC_RBP || (s.norm_mode >= LK_RBP_NORM_SERIES && s.norm_mode <= LK_RBP_NORM_LIST),
                   LK_ERR_INVALID, "lk_rank_metrics: metric %d has unknown RBP normalisation %d", m, s.norm_mode);
    }
    if (a.n_lists == 0 || a.n_metrics == 0) return LK_OK;
    LK_REQUIRE(a.d_rec_indptr && a.d_rec_items && a.d_test_indptr && a.d_test_items && a.d_nrel, LK_ERR_INVALID,
               "lk_rank_metrics: null list or test CSR");
    LK_REQUIRE(a.d_weights && a.d_norms && a.d_out, LK_ERR_INVALID, "lk_rank_metrics: null tables or output");
    LK_REQUIRE(a.n_lists <= (int64_t)INT32_MAX * METRIC_WARPS, LK_ERR_UNSUPPORTED, "lk_rank_metrics: batch too large");

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((a.n_lists + METRIC_WARPS - 1) / METRIC_WARPS);
    rank_metrics_kernel<<<grid, METRIC_WARPS * 32, 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_item_exposure(const lk_item_exposure_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_item_exposure: null args");
    const lk_item_exposure_args &a = *args;
    LK_REQUIRE(a.n_items >= 0 && a.n_entries >= 0, LK_ERR_INVALID, "lk_item_exposure: negative size");
    if (a.n_items == 0) return LK_OK;
    LK_REQUIRE(a.d_totals != nullptr, LK_ERR_INVALID, "lk_item_exposure: null totals");
    LK_REQUIRE(a.n_entries == 0 || (a.d_sorted_items && a.d_order && a.d_entry_list), LK_ERR_INVALID,
               "lk_item_exposure: null entries");
    LK_REQUIRE(a.d_weights == nullptr || a.n_entries == 0 || a.d_entry_rank != nullptr, LK_ERR_INVALID,
               "lk_item_exposure: d_entry_rank is required with d_weights");

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((a.n_items + 255) / 256);
    item_exposure_kernel<<<grid, 256, 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
