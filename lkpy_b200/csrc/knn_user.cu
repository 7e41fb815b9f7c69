// knn_user.cu — user-kNN neighbour search for sm_90a.
//
// Replaces the host step of UserKNNScorer (src/lenskit/knn/user.py:189-214):
//   nbr_sims = user_vectors @ x;  nbr_sims[self] = 0;  keep nbr_sims >= min_sim
// for a batch of sparse query vectors x, with user_vectors in f64.
//
// Bit-exactness contract: SciPy's f64 `csr @ vec` sums each user row in ascending item order — an
// f64 multiply, then an add, no FMA, from +0.0.  Items outside the query only add +-0.0, which cannot
// change a nonzero sum, so sim(q, v) is exactly the sequence
//   acc[v] = acc[v] + VT[i, v] * x[i]      for the query's items i ascending,
// each step rounded on its own (__dmul_rn / __dadd_rn; nvcc would otherwise contract to DFMA).  This is the
// shared tile core (tiles.cuh) over f64 accumulators: the query's items, ascending, are the input rows and
// their VT rows the segments, so every accumulator receives all its additions in ascending item order.  The
// threshold is compared in f64 (a sim just above min_sim whose f32 cast falls below it is kept, as in the
// reference).
//
// Work units are (query, user tile), handed out most-expensive-first from an atomic counter by a
// persistent grid.  The pool epilogue visits every accumulator of the tile: at the ML-25M shape a median
// query makes ~4x more products per tile than the tile has users and ~40 % of all users are neighbours, so
// tracking touched words would skip little; a unit with no products at all (no item of the query reaches
// the tile) skips it.

#include <algorithm>

#include "tiles.cuh"

namespace lk {

constexpr int UKNN_WARPS = 16;
constexpr int UKNN_NT = UKNN_WARPS * 32;
constexpr int UKNN_FIXED_SMEM = UKNN_WARPS * 4 + 16;  // per-warp counts

__global__ void uknn_query_cost_kernel(lk_uknn_search_args a, int64_t *__restrict__ cost)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < a.n_queries; q += warps) {
        long long s = 0;
        for (int64_t p = a.d_q_begin[q] + lane; p < a.d_q_end[q]; p += 32) {
            const int i = a.d_q_items[p];
            s += a.d_vt_indptr[i + 1] - a.d_vt_indptr[i];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
        if (lane == 0) cost[q] = s;
    }
}

__global__ void __launch_bounds__(UKNN_NT, 2) uknn_search_kernel(lk_uknn_search_args a)
{
    constexpr int W = UKNN_WARPS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ int s_work;
    const lk_knn_geom &g = a.geom;
    const int TW = g.tile_cols, S1 = g.n_subtiles + 1, H = g.n_halves;
    const int CW = W * TW;
    double *acc = reinterpret_cast<double *>(smem_raw);  // [CW]
    int *wcnt = reinterpret_cast<int *>(acc + CW);        // [W]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double min_sim = a.min_sim;

    for (int idx = tid; idx < CW; idx += UKNN_NT) acc[idx] = 0.0;
    __syncthreads();

    for (;;) {
        const int64_t wi = cta_next_work(a.d_work_counter, nullptr, &s_work);
        if (wi >= a.n_work) break;
        const int unit = a.d_sched[wi];
        const int q = unit / H, h = unit - q * H;
        const int s = h * W + warp;  // this warp's sub-tile: users [col0, col0 + TW)
        const int col0 = s * TW;
        double *my = acc + warp * TW;

        // products: the query's items in ascending order play the input rows
        const int64_t q0 = a.d_q_begin[q];
        const int m = (int)(a.d_q_end[q] - q0);
        bool any = false;
        for (int t0 = 0; t0 < m; t0 += 32) {
            int len = 0, base = 0;
            double x = 0.0;
            if (t0 + lane < m) {
                const int i = __ldg(a.d_q_items + q0 + t0 + lane);
                x = __ldg(a.d_q_vals + q0 + t0 + lane);
                const int32_t *tp = a.d_tile_ptr + (size_t)i * S1 + s;
                base = __ldg(tp);
                len = __ldg(tp + 1) - base;
            }
            any |= warp_walk_segments(base, len, lane, [&](bool valid, int own, int src) {
                const double xq = __shfl_sync(FULL, x, own);
                int j = 0;
                double prod = 0.0;
                if (valid) {
                    j = __ldg(a.d_vt_users + src) - col0;
                    prod = __dmul_rn(__ldg(a.d_vt_vals + src), xq);  // VT[i,v] * x[i], never contracted
                }
                warp_apply_in_owner_order(valid, own, [&] { my[j] = __dadd_rn(my[j], prod); });
            });
        }
        if (!__syncthreads_or(any)) {  // no item of the query reaches this tile: every accumulator is still +0.0
            if (tid == 0) {
                a.d_part_cnt[unit] = 0;
                a.d_pool_off[unit] = 0;
            }
            continue;
        }

        // epilogue: one pool segment per unit in user order; the threshold is compared in f64, and the kept sims
        // are rounded to nearest, as NumPy's astype(float32)
        const int self = a.d_q_self != nullptr ? a.d_q_self[q] : -1;
        cta_emit_pool_segment<W>(
            my, TW, col0, unit, [&](double sim, int v) { return sim >= min_sim && v != self; },
            [](double sim, int) { return __float_as_uint((float)sim); }, 0.0, wcnt, a.d_pool_cursor, a.pool_capacity,
            a.d_status, a.d_pool_off, a.d_part_cnt, a.d_pool_rows, reinterpret_cast<uint32_t *>(a.d_pool_sims));
    }
}

static int uknn_smem_bytes(const lk_knn_geom &g) { return g.warps * g.tile_cols * 8 + UKNN_FIXED_SMEM; }

}  // namespace lk

using namespace lk;

extern "C" {

int lk_uknn_geometry(int32_t n_users, int32_t n_items, int32_t ctas_per_sm, lk_knn_geom *geom)
{
    LK_REQUIRE(geom != nullptr && n_users >= 1 && n_items >= 0, LK_ERR_INVALID, "lk_uknn_geometry: bad arguments");
    const int ctas = ctas_per_sm > 0 ? ctas_per_sm : 2;
    LK_REQUIRE(ctas <= 2, LK_ERR_INVALID, "lk_uknn_geometry: ctas_per_sm must be 0, 1 or 2");
    // 8-byte accumulators over the users; VT's rows (items) are the input rows
    tile_geometry(n_items, n_users, UKNN_WARPS, ctas, 8, UKNN_FIXED_SMEM, 64, geom);
    return LK_OK;
}

static int uknn_check(const lk_uknn_search_args *args, const char *who)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "%s: null args", who);
    const lk_uknn_search_args &a = *args;
    LK_REQUIRE(a.n_queries >= 0 && (int64_t)a.n_queries * a.geom.n_halves < 0x7fffffffLL, LK_ERR_INVALID,
               "%s: n_queries * n_halves must be < 2^31", who);
    LK_REQUIRE(a.geom.warps == UKNN_WARPS && a.geom.n_halves >= 1, LK_ERR_INVALID,
               "%s: geometry not from lk_uknn_geometry", who);
    if (a.n_queries > 0)
        LK_REQUIRE(a.d_q_begin && a.d_q_end && a.d_q_items && a.d_vt_indptr, LK_ERR_INVALID, "%s: null query", who);
    return LK_OK;
}

int lk_uknn_query_cost(const lk_uknn_search_args *args, int64_t *d_cost, void *stream)
{
    if (int rc = uknn_check(args, "lk_uknn_query_cost")) return rc;
    if (args->n_queries == 0) return LK_OK;
    LK_REQUIRE(d_cost != nullptr, LK_ERR_INVALID, "lk_uknn_query_cost: null cost");
    uknn_query_cost_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, d_cost);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_uknn_search(const lk_uknn_search_args *args, void *stream)
{
    if (int rc = uknn_check(args, "lk_uknn_search")) return rc;
    const lk_uknn_search_args &a = *args;
    LK_REQUIRE(a.d_work_counter && a.d_status && a.d_pool_cursor, LK_ERR_INVALID, "lk_uknn_search: null counter");
    LK_REQUIRE(a.min_sim > 0.0, LK_ERR_INVALID, "lk_uknn_search: min_sim must be positive");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_status, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
    if (a.n_work == 0) return LK_OK;
    LK_REQUIRE(a.d_vt_users && a.d_vt_vals && a.d_tile_ptr && a.d_q_vals && a.d_sched && a.d_pool_rows &&
                   a.d_pool_sims && a.d_pool_off && a.d_part_cnt,
               LK_ERR_INVALID, "lk_uknn_search: null pointer");
    const int smem = uknn_smem_bytes(a.geom);
    int64_t grid = (int64_t)sm_count() * a.geom.ctas_per_sm;
    if (grid > a.n_work) grid = a.n_work;
    LK_CUDA_TRY(cudaFuncSetAttribute(uknn_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    uknn_search_kernel<<<(unsigned)grid, UKNN_NT, smem, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_uknn_pool_to_csr(const lk_uknn_search_args *args, const int64_t *d_out_indptr, int32_t *d_out_rows,
                        float *d_out_sims, void *stream)
{
    if (int rc = uknn_check(args, "lk_uknn_pool_to_csr")) return rc;
    if (args->n_queries == 0) return LK_OK;
    LK_REQUIRE(d_out_indptr && d_out_rows && d_out_sims && args->d_pool_off && args->d_part_cnt, LK_ERR_INVALID,
               "lk_uknn_pool_to_csr: null pointer");
    const lk_uknn_search_args &a = *args;
    return launch_pool_to_csr(a.n_queries, a.geom.n_halves, a.d_pool_off, a.d_part_cnt, a.d_pool_rows, a.d_pool_sims,
                              d_out_indptr, d_out_rows, d_out_sims, stream);
}

}  // extern "C"
