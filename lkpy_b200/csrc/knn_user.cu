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
// each step rounded on its own (__dmul_rn / __dadd_rn; nvcc would otherwise contract to DFMA).  The
// structure is the item-kNN build's (knn_build.cu) with the roles swapped: the query's items play the
// build's users, VT rows play UI rows, and one warp owns a contiguous user sub-tile of f64 accumulators
// in shared memory, so every accumulator receives all its additions from one warp in ascending item
// order.  The threshold is compared in f64 (a sim just above min_sim whose f32 cast falls below it is
// kept, as in the reference).
//
// Work units are (query, user tile), handed out most-expensive-first from an atomic counter by a
// persistent grid.  After a unit's products, each warp scans its own sub-tile 32 accumulators at a time
// (ballot + popcount keep user order), the CTA bump-allocates one pool segment for the unit, the warps
// write their survivors into it and reset the accumulators.  The scan visits every accumulator of the
// tile: at the ML-25M shape a median query makes ~4x more products per tile than the tile has users and
// ~40 % of all users are neighbours, so tracking touched words would skip little; a unit with no
// products at all (no item of the query reaches the tile) skips the scan.

#include <algorithm>

#include "common.cuh"

namespace lk {

constexpr int UKNN_WARPS = 16;
constexpr int UKNN_NT = UKNN_WARPS * 32;

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
    __shared__ int64_t s_work;
    __shared__ unsigned long long s_off;
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
        if (tid == 0) s_work = fetch_work(a.d_work_counter, nullptr);
        __syncthreads();
        const int64_t wi = s_work;
        __syncthreads();
        if (wi >= a.n_work) break;
        const int unit = a.d_sched[wi];
        const int q = unit / H, h = unit - q * H;
        const int s = h * W + warp;  // this warp's sub-tile: users [col0, col0 + TW)
        const int col0 = s * TW;
        double *my = acc + warp * TW;

        // ------------------------------------------------------------------
        // products: the query's items in ascending order, 32 at a time flattened over the lanes for the
        // loads, applied one item per round (the lanes of one item hit distinct users)
        // ------------------------------------------------------------------
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
            const int incl = warp_incl_scan(len, lane);
            const int total = __shfl_sync(FULL, incl, 31);
            any |= total > 0;
            const int adj = base - (incl - len);  // source index = adj[owner] + e
            for (int e0 = 0; e0 < total; e0 += 32) {
                const int e = e0 + lane;
                const bool valid = e < total;
                int own = 0;  // owner: smallest lane with incl > e
#pragma unroll
                for (int step = 16; step > 0; step >>= 1) {
                    const int t = __shfl_sync(FULL, incl, own + step - 1);
                    if (t <= e) own += step;
                }
                own = min(own, 31);
                const int src = __shfl_sync(FULL, adj, own) + e;
                const double xq = __shfl_sync(FULL, x, own);
                int j = 0;
                double prod = 0.0;
                if (valid) {
                    j = __ldg(a.d_vt_users + src) - col0;
                    prod = __dmul_rn(__ldg(a.d_vt_vals + src), xq);  // VT[i,v] * x[i], never contracted
                }
                unsigned pend = __ballot_sync(FULL, valid);
                while (pend) {
                    const int leader = __ffs(pend) - 1;
                    const int oo = __shfl_sync(FULL, own, leader);
                    const bool mine = valid && own == oo;
                    if (mine) my[j] = __dadd_rn(my[j], prod);
                    __syncwarp();
                    pend &= ~__ballot_sync(FULL, mine);
                }
            }
        }
        if (!__syncthreads_or(any)) {  // no item of the query reaches this tile: every accumulator is still +0.0
            if (tid == 0) {
                a.d_part_cnt[unit] = 0;
                a.d_pool_off[unit] = 0;
            }
            continue;
        }

        // ------------------------------------------------------------------
        // epilogue: count, one pool segment per unit, write in user order, reset
        // ------------------------------------------------------------------
        const int self = a.d_q_self != nullptr ? a.d_q_self[q] : -1;
        int cnt = 0;
        for (int c0 = 0; c0 < TW; c0 += 32) {
            const int v = col0 + c0 + lane;
            const bool keep = my[c0 + lane] >= min_sim && v != self;
            cnt += __popc(__ballot_sync(FULL, keep));
        }
        if (lane == 0) wcnt[warp] = cnt;
        __syncthreads();
        if (tid == 0) {
            int n = 0;
            for (int w = 0; w < W; w++) n += wcnt[w];
            unsigned long long off = atomicAdd(a.d_pool_cursor, (unsigned long long)n);
            if (off + (unsigned long long)n > (unsigned long long)a.pool_capacity) {
                atomicCAS(a.d_status, 0, 1);
                off = ~0ull;
            }
            s_off = off;
            a.d_pool_off[unit] = (int64_t)off;
            a.d_part_cnt[unit] = n;
        }
        __syncthreads();
        const unsigned long long off = s_off;
        int pos = 0;
        for (int w = 0; w < warp; w++) pos += wcnt[w];
        for (int c0 = 0; c0 < TW; c0 += 32) {
            const int v = col0 + c0 + lane;
            const double sim = my[c0 + lane];
            const bool keep = sim >= min_sim && v != self;
            const unsigned b = __ballot_sync(FULL, keep);
            if (keep && off != ~0ull) {
                const unsigned long long k = off + pos + __popc(b & ((1u << lane) - 1u));
                a.d_pool_rows[k] = v;
                a.d_pool_sims[k] = (float)sim;  // round to nearest, as NumPy's astype(float32)
            }
            pos += __popc(b);
            my[c0 + lane] = 0.0;
        }
        __syncthreads();  // wcnt and s_off are rewritten by the next unit
    }
}

__global__ void uknn_pool_to_csr_kernel(lk_uknn_search_args a, const int64_t *__restrict__ out_indptr,
                                        int32_t *__restrict__ out_rows, float *__restrict__ out_sims)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t H = a.geom.n_halves;
    for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < a.n_queries; q += warps)
        warp_copy_pool_segments(q * H, (q + 1) * H, a.d_pool_off, a.d_part_cnt, a.d_pool_rows, a.d_pool_sims,
                                out_indptr[q], out_rows, out_sims, lane);
}

static int uknn_smem_bytes(const lk_knn_geom &g) { return g.warps * g.tile_cols * 8 + g.warps * 4 + 16; }

}  // namespace lk

using namespace lk;

extern "C" {

int lk_uknn_geometry(int32_t n_users, int32_t n_items, int32_t ctas_per_sm, lk_knn_geom *geom)
{
    LK_REQUIRE(geom != nullptr && n_users >= 1 && n_items >= 0, LK_ERR_INVALID, "lk_uknn_geometry: bad arguments");
    const int warps = UKNN_WARPS;
    const int ctas = ctas_per_sm > 0 ? ctas_per_sm : 2;
    LK_REQUIRE(ctas <= 2, LK_ERR_INVALID, "lk_uknn_geometry: ctas_per_sm must be 0, 1 or 2");
    // shared memory budget per CTA (227 KB usable per SM, 1 KB reserved per CTA), 8-byte accumulators
    const int budget = (227 * 1024) / ctas - 1024 - (warps * 4 + 16) - 64;
    const int max_cols = budget / 8;
    int halves = (n_users + max_cols - 1) / max_cols;
    if (halves < 1) halves = 1;
    const int cw = (n_users + halves - 1) / halves;
    int tw = (cw + warps - 1) / warps;
    tw = (tw + 31) & ~31;
    while ((int64_t)tw * warps > max_cols && tw > 32) tw -= 32;
    halves = (n_users + tw * warps - 1) / (tw * warps);
    geom->n_users = n_items;  // VT rows
    geom->n_items = n_users;  // accumulator columns
    geom->warps = warps;
    geom->tile_cols = tw;
    geom->n_halves = halves;
    geom->n_subtiles = halves * warps;
    geom->smem_bytes = uknn_smem_bytes(*geom);
    geom->ctas_per_sm = ctas;
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
    uknn_pool_to_csr_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, d_out_indptr,
                                                                                        d_out_rows, d_out_sims);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
