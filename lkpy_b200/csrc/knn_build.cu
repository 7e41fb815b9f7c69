// knn_build.cu — item-item similarity build for sm_90a.
//
// Replaces src/accel/knn/item_train.rs:65-152 (ItemSimTask::invoke, sim_row):
// row i of IU * UI by Gustavson accumulation, `>= min_sim` filter, optional
// stable top-`save_nbrs` truncation, rows returned sorted by column.
//
// Bit-exactness contract (SURVEY.md §7): for every output pair (i, j) the
// reference adds fl(r_iu * r_uj) into dots[j] over the common users u in
// ascending order, starting from +0.0f, with no FMA contraction.  This kernel
// reproduces exactly that sequence of roundings:
//   * one warp owns one accumulator sub-tile (a contiguous column range) of
//     the row in shared memory, so all updates of a given dots[j] come from one
//     warp, which walks the item's users in ascending order;
//   * inside a warp the products of up to 32 users are flattened across the
//     lanes for the loads, then applied user by user (ascending), lanes of one
//     user touching distinct columns;
//   * products use __fmul_rn / __fadd_rn.
// The truncation order is the reference's stable sort by similarity over the
// first-touch order, i.e. (sim desc, first common user asc, column asc); the
// first common user is only needed to cut a tie group at the K-th place and is
// then recovered by intersecting the two items' user lists.
//
// The work is HBM/L2-streaming integer+f32 scatter work (8 B per product), not
// a GEMM: no tensor cores.  Layout: a CTA of W warps holds W sub-tiles (one
// "column half" of the row); an item row takes n_halves passes.  Work units
// (item, half, piece) are pulled most-expensive-first from an atomic counter by a
// persistent grid; `piece` cuts the unit of a very expensive item into column
// slices (piece p of P: the p-th P-th of every warp's sub-tile) so that one hot
// item cannot keep a single CTA busy longer than a GPU's fair share of the whole
// build — a column split leaves every dots[j] with its full ascending-user sum
// (a user split would change the rounding).
//
// Ordering inside a warp: the products of up to 32 users are flattened over the
// lanes in (user, column) order and applied one user per round (the lanes of one
// user hit distinct columns).

#include <algorithm>
#include <cstdlib>

#include "common.cuh"

namespace lk {

constexpr uint32_t SENT = 0xffffffffu;  // "never touched" accumulator marker (a NaN no product yields)
constexpr int HIST_BINS = 2048;

__device__ __forceinline__ bool is_cand(uint32_t bits, float min_sim)
{
    return bits != SENT && __uint_as_float(bits) >= min_sim;
}

// ---------------------------------------------------------------------------
// CTA-wide radix select: the kk-th largest 32-bit key among the valid elements
// of an index space [0, n).  get(idx, key) returns validity.  On return
// *theta = that key, *need = how many elements equal to theta still belong to
// the top-kk (1 <= need <= count(== theta)), *n_eq = count(== theta).
// hist: HIST_BINS uint32 in shared memory; bc: 4 ints of shared broadcast space.
// All threads of the CTA must call; contains __syncthreads.
// ---------------------------------------------------------------------------
template <typename Get>
__device__ void cta_select_kth_largest(Get get, int n, int kk, uint32_t *hist, int *bc,
                                       uint32_t *theta, int *need, int *n_eq)
{
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
    uint32_t prefix = 0, mask = 0;
#pragma unroll
    for (int pass = 0; pass < 3; pass++) {
        const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0;
        const int nb = pass == 2 ? 1024 : 2048;
        for (int b = tid; b < HIST_BINS; b += nt) hist[b] = 0;
        __syncthreads();
        for (int idx = tid; idx < n; idx += nt) {
            uint32_t key;
            if (get(idx, key) && (key & mask) == prefix) atomicAdd(&hist[(key >> shift) & (nb - 1)], 1u);
        }
        __syncthreads();
        if (tid < 32) {
            const int per = nb / 32;  // bins per lane, lane 0 holds the top bins
            const int top = nb - lane * per;
            uint32_t s = 0;
            for (int b = top - per; b < top; b++) s += hist[b];
            uint32_t cum = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(FULL, cum, o);
                if (lane >= o) cum += t;
            }
            const unsigned hit = __ballot_sync(FULL, cum >= (uint32_t)kk);
            const int first = __ffs(hit) - 1;
            if (lane == first) {
                uint32_t run = cum - s;
                int d = top - 1;
                for (; d >= top - per; d--) {
                    run += hist[d];
                    if (run >= (uint32_t)kk) break;
                }
                bc[0] = d;
                bc[1] = (int)(run - hist[d]);  // elements strictly above digit d
                bc[2] = (int)hist[d];
            }
        }
        __syncthreads();
        prefix |= (uint32_t)bc[0] << shift;
        mask |= (uint32_t)(nb - 1) << shift;
        kk -= bc[1];
        *n_eq = bc[2];
        __syncthreads();
    }
    *theta = prefix;
    *need = kk;
}

// smallest common user of items i and j (both rows of IU sorted ascending)
__device__ int first_common_user(const int32_t *__restrict__ iu_indptr,
                                 const int32_t *__restrict__ iu_cols, int i, int j)
{
    int a0 = iu_indptr[i], a1 = iu_indptr[i + 1];
    int b0 = iu_indptr[j], b1 = iu_indptr[j + 1];
    if (a1 - a0 > b1 - b0) {
        int t = a0; a0 = b0; b0 = t;
        t = a1; a1 = b1; b1 = t;
    }
    for (int p = a0; p < a1; p++) {  // shorter list ascending
        const int u = iu_cols[p];
        int lo = b0, hi = b1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (iu_cols[mid] < u) lo = mid + 1; else hi = mid;
        }
        if (lo < b1 && iu_cols[lo] == u) return u;
        b0 = lo;  // later users cannot sit before this point
    }
    return 0x7fffffff;
}

__global__ void tile_ptr_kernel(lk_knn_geom g, const int32_t *__restrict__ ui_indptr,
                                const int32_t *__restrict__ ui_cols, int32_t *__restrict__ tptr)
{
    const int64_t S1 = g.n_subtiles + 1;
    const int64_t total = (int64_t)g.n_users * S1;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int u = (int)(idx / S1), s = (int)(idx % S1);
        const int64_t bound = (int64_t)s * g.tile_cols;
        int lo = ui_indptr[u], hi = ui_indptr[u + 1];
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((int64_t)ui_cols[mid] < bound) lo = mid + 1; else hi = mid;
        }
        tptr[idx] = lo;
    }
}

__global__ void row_cost_kernel(int n_items, const int32_t *__restrict__ ui_indptr,
                                const int32_t *__restrict__ iu_indptr,
                                const int32_t *__restrict__ iu_cols, int64_t *__restrict__ cost)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_items; i += warps) {
        long long s = 0;
        for (int p = iu_indptr[i] + lane; p < iu_indptr[i + 1]; p += 32) {
            const int u = iu_cols[p];
            s += ui_indptr[u + 1] - ui_indptr[u];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
        if (lane == 0) cost[i] = s;
    }
}

template <int W>
__global__ void __launch_bounds__(W * 32, 1024 / (W * 32)) knn_build_kernel(lk_knn_build_args a)
{
    constexpr int NT = W * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const lk_knn_geom &g = a.geom;
    const int TW = g.tile_cols, S1 = g.n_subtiles + 1;
    const int CW = W * TW;
    uint32_t *acc = reinterpret_cast<uint32_t *>(smem_raw);       // [CW] f32 bit patterns
    uint32_t *hist = acc + CW;                                     // [HIST_BINS]
    int *bc = reinterpret_cast<int *>(hist + HIST_BINS);           // [16]
    int *wsum = bc + 16;                                           // [W]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = a.save_nbrs;
    const float min_sim = a.min_sim;
    int32_t *tie_cols = a.d_tie_scratch + (size_t)blockIdx.x * 2 * CW;
    int32_t *tie_fu = tie_cols + CW;

    for (int idx = tid; idx < CW; idx += NT) acc[idx] = SENT;
    __syncthreads();

    const int64_t n_work = a.n_work;
    for (;;) {
        if (tid == 0) bc[8] = fetch_work(a.d_work_counter, a.d_cancel);
        __syncthreads();
        const int64_t wi = bc[8];
        __syncthreads();
        if (wi >= n_work) break;
        const int uid = a.d_sched[wi];
        const int4 un = __ldg(reinterpret_cast<const int4 *>(a.d_units) + uid);
        const int item = un.x, h = un.y;
        const int pw = TW / un.w;  // columns of this piece inside every warp's sub-tile

        // ------------------------------------------------------------------
        // accumulate: warp `warp` owns columns [col0, col0 + TW), of which this unit covers [jlo, jhi)
        // ------------------------------------------------------------------
        {
            const int s = h * W + warp;
            const int col0 = s * TW;
            const int jlo = un.z * pw, jhi = jlo + pw;
            uint32_t *my = acc + warp * TW;
            const int iu0 = a.d_iu_indptr[item];
            const int m = a.d_iu_indptr[item + 1] - iu0;
            for (int t0 = 0; t0 < m; t0 += 32) {
                int len = 0, base = 0;
                float r = 0.0f;
                if (t0 + lane < m) {
                    const int u = __ldg(a.d_iu_cols + iu0 + t0 + lane);
                    r = __ldg(a.d_iu_vals + iu0 + t0 + lane);
                    const int32_t *tp = a.d_tile_ptr + (size_t)u * S1 + s;
                    base = __ldg(tp);
                    len = __ldg(tp + 1) - base;
                }
                const int incl = warp_incl_scan(len, lane);
                const int total = __shfl_sync(FULL, incl, 31);
                const int adj = base - (incl - len);  // source index = adj[owner] + e
                for (int e0 = 0; e0 < total; e0 += 32) {
                    const int e = e0 + lane;
                    bool valid = e < total;
                    int q = 0;  // owner: smallest lane with incl > e
#pragma unroll
                    for (int step = 16; step > 0; step >>= 1) {
                        const int t = __shfl_sync(FULL, incl, q + step - 1);
                        if (t <= e) q += step;
                    }
                    q = min(q, 31);
                    const int src = __shfl_sync(FULL, adj, q) + e;
                    const float rq = __shfl_sync(FULL, r, q);
                    int j = 0;
                    float prod = 0.0f;
                    if (valid) {
                        const int col = __ldg(a.d_ui_cols + src);
                        const float val = __ldg(a.d_ui_vals + src);
                        prod = __fmul_rn(rq, val);  // never contracted (item_train.rs:128)
                        j = col - col0;
                        // diagonal excluded by index (item_train.rs:120-122); columns of other pieces are not ours
                        valid = col != item && j >= jlo && j < jhi;
                    }
                    // users in ascending order, one user per round: the lanes of one user hit distinct columns.
                    // (Grouping lanes by column instead — __match_any_sync, or one ballot per column bit — was
                    // measured slower on ML-25M-shaped data: a popular column is present in most users'
                    // segments, so the rounds per batch stay near the number of users.)
                    unsigned pend = __ballot_sync(FULL, valid);
                    while (pend) {
                        const int leader = __ffs(pend) - 1;
                        const int qq = __shfl_sync(FULL, q, leader);
                        const bool mine = valid && q == qq;
                        if (mine) {
                            const uint32_t old = my[j];
                            const float b = old == SENT ? 0.0f : __uint_as_float(old);
                            my[j] = __float_as_uint(__fadd_rn(b, prod));
                        }
                        __syncwarp();
                        pend &= ~__ballot_sync(FULL, mine);
                    }
                }
            }
        }
        __syncthreads();

        // ------------------------------------------------------------------
        // epilogue: threshold, (top-K | all), emit, reset accumulators
        // ------------------------------------------------------------------
        const int half_col0 = h * CW;
        const int64_t pidx = uid;  // partial lists / pool segments are indexed by unit
        // candidate count
        int local = 0;
        for (int idx = tid; idx < CW; idx += NT) local += is_cand(acc[idx], min_sim) ? 1 : 0;
        // block reduce of `local`
        {
            int v = local;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
            if (lane == 0) wsum[warp] = v;
        }
        __syncthreads();
        int n_cand = 0;
        for (int w = 0; w < W; w++) n_cand += wsum[w];
        __syncthreads();

        if (K <= 0) {
            // unbounded: all candidates, in column order, into the pool
            if (tid == 0) {
                unsigned long long off = atomicAdd(a.d_pool_cursor, (unsigned long long)n_cand);
                if (off + (unsigned long long)n_cand > (unsigned long long)a.pool_capacity) {
                    atomicCAS(a.d_status, 0, 1);
                    off = ~0ull;
                }
                reinterpret_cast<unsigned long long *>(bc)[0] = off;
                a.d_pool_off[pidx] = (int64_t)off;
                a.d_part_cnt[pidx] = n_cand;
            }
            __syncthreads();
            const unsigned long long off = reinterpret_cast<unsigned long long *>(bc)[0];
            // contiguous column range per thread keeps column order
            const int per = (CW + NT - 1) / NT;
            const int c_lo = min(CW, tid * per), c_hi = min(CW, c_lo + per);
            int cnt = 0;
            for (int c = c_lo; c < c_hi; c++) cnt += is_cand(acc[c], min_sim) ? 1 : 0;
            const int incl = warp_incl_scan(cnt, lane);
            if (lane == 31) wsum[warp] = incl;
            __syncthreads();
            int woff = 0;
            for (int w = 0; w < warp; w++) woff += wsum[w];
            int pos = woff + incl - cnt;
            if (off != ~0ull) {
                for (int c = c_lo; c < c_hi; c++) {
                    const uint32_t bits = acc[c];
                    if (is_cand(bits, min_sim)) {
                        a.d_pool_cols[off + pos] = half_col0 + c;
                        a.d_pool_vals[off + pos] = __uint_as_float(bits);
                        pos++;
                    }
                }
            }
            __syncthreads();
            for (int idx = tid; idx < CW; idx += NT) acc[idx] = SENT;
            __syncthreads();
            continue;
        }

        int32_t *pc = a.d_part_cols + pidx * K;
        float *pv = a.d_part_vals + pidx * K;
        if (n_cand <= K) {
            if (tid == 0) {
                bc[4] = 0;
                a.d_part_cnt[pidx] = n_cand;
            }
            __syncthreads();
            for (int idx = tid; idx < CW; idx += NT) {
                const uint32_t bits = acc[idx];
                if (is_cand(bits, min_sim)) {
                    const int slot = atomicAdd(&bc[4], 1);
                    pc[slot] = half_col0 + idx;
                    pv[slot] = __uint_as_float(bits);
                }
                acc[idx] = SENT;
            }
            __syncthreads();
            continue;
        }

        // K-th largest similarity of this half
        uint32_t theta;
        int need, n_eq;
        cta_select_kth_largest(
            [&](int idx, uint32_t &key) {
                key = acc[idx];
                return is_cand(key, min_sim);
            },
            CW, K, hist, bc, &theta, &need, &n_eq);
        const bool cut = n_eq > need;  // the tie group at theta does not fit entirely
        if (tid == 0) {
            bc[4] = 0;  // list slots
            bc[5] = 0;  // tie slots
            a.d_part_cnt[pidx] = K;
        }
        __syncthreads();
        for (int idx = tid; idx < CW; idx += NT) {
            const uint32_t bits = acc[idx];
            if (is_cand(bits, min_sim)) {
                if (bits > theta || (bits == theta && !cut)) {
                    const int slot = atomicAdd(&bc[4], 1);
                    pc[slot] = half_col0 + idx;
                    pv[slot] = __uint_as_float(bits);
                } else if (bits == theta) {
                    const int slot = atomicAdd(&bc[5], 1);
                    tie_cols[slot] = half_col0 + idx;
                }
            }
            acc[idx] = SENT;
        }
        __syncthreads();
        if (cut) {
            // cut the tie group by (first common user asc, column asc)
            const int G = bc[5];
            const int base_slot = bc[4];
            for (int t = tid; t < G; t += NT)
                tie_fu[t] = first_common_user(a.d_iu_indptr, a.d_iu_cols, item, tie_cols[t]);
            __syncthreads();
            // need-th smallest first-user: select on inverted keys
            uint32_t th_fu_inv;
            int need_fu, eq_fu;
            cta_select_kth_largest(
                [&](int t, uint32_t &key) {
                    key = ~(uint32_t)tie_fu[t];
                    return true;
                },
                G, need, hist, bc, &th_fu_inv, &need_fu, &eq_fu);
            const int th_fu = (int)~th_fu_inv;
            // among fu == th_fu keep the need_fu smallest columns
            uint32_t th_col_inv = 0;
            int need_col, eq_col;
            cta_select_kth_largest(
                [&](int t, uint32_t &key) {
                    key = ~(uint32_t)tie_cols[t];
                    return tie_fu[t] == th_fu;
                },
                G, need_fu, hist, bc, &th_col_inv, &need_col, &eq_col);
            const int th_col = (int)~th_col_inv;
            if (tid == 0) bc[6] = 0;
            __syncthreads();
            for (int t = tid; t < G; t += NT) {
                const int fu = tie_fu[t], col = tie_cols[t];
                if (fu < th_fu || (fu == th_fu && col <= th_col)) {
                    const int slot = base_slot + atomicAdd(&bc[6], 1);
                    pc[slot] = col;
                    pv[slot] = __uint_as_float(theta);
                }
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------
// merge the per-half top-K lists: one CTA (128 threads) per item
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) knn_merge_kernel(lk_knn_build_args a, int32_t *__restrict__ out_cols,
                                                       float *__restrict__ out_vals,
                                                       int32_t *__restrict__ out_cnt)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int K = a.save_nbrs;
    const int cap = a.max_units_per_item * K;
    int32_t *cols = reinterpret_cast<int32_t *>(smem_raw);
    float *sims = reinterpret_cast<float *>(cols + cap);
    int32_t *fus = reinterpret_cast<int32_t *>(sims + cap);
    int32_t *state = fus + cap;  // 0 drop, 1 keep, 2 tie group
    __shared__ int s_n, s_gt, s_keep;
    const int tid = threadIdx.x;
    for (int item = blockIdx.x; item < a.geom.n_items; item += gridDim.x) {
        const int u0 = a.d_unit_ptr[item], u1 = a.d_unit_ptr[item + 1];
        if (tid == 0) {
            int n = 0;
            for (int u = u0; u < u1; u++) n += a.d_part_cnt[u];
            s_n = n;
            s_keep = 0;
        }
        __syncthreads();
        const int n = s_n;
        // gather
        {
            int off = 0;
            for (int u = u0; u < u1; u++) {
                const int c = a.d_part_cnt[u];
                for (int t = tid; t < c; t += blockDim.x) {
                    cols[off + t] = a.d_part_cols[(int64_t)u * K + t];
                    sims[off + t] = a.d_part_vals[(int64_t)u * K + t];
                }
                off += c;
            }
        }
        __syncthreads();
        // classify by similarity rank
        for (int e = tid; e < n; e += blockDim.x) {
            const float s = sims[e];
            int gt = 0, eq = 0;
            for (int f = 0; f < n; f++) {
                gt += sims[f] > s;
                eq += sims[f] == s;
            }
            int st = 0;
            if (gt + eq <= K) st = 1;
            else if (gt < K) st = 2;
            state[e] = st;
            fus[e] = gt;  // reused: number strictly greater (same for the whole tie group)
        }
        __syncthreads();
        // tie group cut: (first common user, column) ascending
        for (int e = tid; e < n; e += blockDim.x)
            if (state[e] == 2) {
                s_gt = fus[e];
            }
        __syncthreads();
        const int gt_grp = s_gt;
        __syncthreads();
        for (int e = tid; e < n; e += blockDim.x)
            if (state[e] == 2) fus[e] = first_common_user(a.d_iu_indptr, a.d_iu_cols, item, cols[e]);
        __syncthreads();
        for (int e = tid; e < n; e += blockDim.x)
            if (state[e] == 2) {
                int r = 0;
                for (int f = 0; f < n; f++)
                    if (state[f] >= 2 && f != e)
                        r += (fus[f] < fus[e]) || (fus[f] == fus[e] && cols[f] < cols[e]);
                // state 3 marks "tie, kept"; other ties keep reading state>=2 consistently
                if (gt_grp + r < K) state[e] = 3;
            }
        __syncthreads();
        // output position = rank by column among kept entries
        for (int e = tid; e < n; e += blockDim.x) {
            const bool keep = state[e] == 1 || state[e] == 3;
            if (keep) {
                int pos = 0;
                for (int f = 0; f < n; f++)
                    pos += (state[f] == 1 || state[f] == 3) && cols[f] < cols[e];
                out_cols[(int64_t)item * K + pos] = cols[e];
                out_vals[(int64_t)item * K + pos] = sims[e];
                atomicAdd(&s_keep, 1);
            }
        }
        __syncthreads();
        if (tid == 0) out_cnt[item] = s_keep;
        __syncthreads();
    }
}

__global__ void pool_to_csr_kernel(lk_knn_build_args a, const int64_t *__restrict__ out_indptr,
                                   int32_t *__restrict__ out_cols, float *__restrict__ out_vals)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int item = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < a.geom.n_items; item += warps) {
        int64_t dst = out_indptr[item];
        // unbounded mode has one unit per (item, half), in column order
        for (int u = a.d_unit_ptr[item]; u < a.d_unit_ptr[item + 1]; u++) {
            const int64_t src = a.d_pool_off[u];
            const int c = a.d_part_cnt[u];
            for (int t = lane; t < c; t += 32) {
                out_cols[dst + t] = a.d_pool_cols[src + t];
                out_vals[dst + t] = a.d_pool_vals[src + t];
            }
            dst += c;
        }
    }
}

static int knn_smem_bytes(const lk_knn_geom &g)
{
    return g.warps * g.tile_cols * 4 + HIST_BINS * 4 + 16 * 4 + g.warps * 4 + 16;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_knn_geometry(int32_t n_users, int32_t n_items, lk_knn_geom *geom)
{
    LK_REQUIRE(geom != nullptr && n_users >= 0 && n_items >= 1, LK_ERR_INVALID,
               "lk_knn_geometry: bad arguments");
    int warps = 16, ctas = 2;
    if (options().knn_warps > 0) warps = options().knn_warps;
    if (options().knn_ctas > 0) ctas = options().knn_ctas;
    LK_REQUIRE(warps == 8 || warps == 16 || warps == 32, LK_ERR_INVALID, "LK_KNN_WARPS must be 8, 16 or 32");
    LK_REQUIRE(ctas >= 1 && ctas <= 8, LK_ERR_INVALID, "LK_KNN_CTAS must be 1..8");
    // shared memory budget per CTA (227 KB usable per SM, 1 KB reserved per CTA)
    const int budget = (227 * 1024) / ctas - 1024 - (HIST_BINS * 4 + 16 * 4 + warps * 4 + 16);
    const int max_cols = budget / 4;
    int halves = (n_items + max_cols - 1) / max_cols;
    if (halves < 1) halves = 1;
    int cw = (n_items + halves - 1) / halves;
    int tw = (cw + warps - 1) / warps;
    tw = (tw + 31) & ~31;
    while ((int64_t)tw * warps > max_cols && tw > 32) tw -= 32;
    halves = (n_items + tw * warps - 1) / (tw * warps);
    geom->n_users = n_users;
    geom->n_items = n_items;
    geom->warps = warps;
    geom->tile_cols = tw;
    geom->n_halves = halves;
    geom->n_subtiles = halves * warps;
    geom->smem_bytes = knn_smem_bytes(*geom);
    geom->ctas_per_sm = ctas;
    return LK_OK;
}

int lk_knn_tile_pointers(const lk_knn_geom *geom, const int32_t *d_ui_indptr,
                         const int32_t *d_ui_cols, int32_t *d_tile_ptr, void *stream)
{
    LK_REQUIRE(geom && d_ui_indptr && d_tile_ptr, LK_ERR_INVALID, "lk_knn_tile_pointers: null");
    if (geom->n_users == 0) return LK_OK;
    tile_ptr_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*geom, d_ui_indptr,
                                                                                  d_ui_cols, d_tile_ptr);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_knn_row_cost(const lk_knn_geom *geom, const int32_t *d_ui_indptr, const int32_t *d_iu_indptr,
                    const int32_t *d_iu_cols, int64_t *d_cost, void *stream)
{
    LK_REQUIRE(geom && d_ui_indptr && d_iu_indptr && d_cost, LK_ERR_INVALID, "lk_knn_row_cost: null");
    row_cost_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        geom->n_items, d_ui_indptr, d_iu_indptr, d_iu_cols, d_cost);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

static int64_t knn_grid(const lk_knn_geom &g, int64_t n_work)
{
    int64_t grid = (int64_t)sm_count() * g.ctas_per_sm;
    if (grid > n_work) grid = n_work;
    return grid < 1 ? 1 : grid;
}

int64_t lk_knn_tie_scratch_ints(const lk_knn_geom *geom)
{
    if (!geom) return -1;
    return (int64_t)sm_count() * geom->ctas_per_sm * 2 * geom->warps * geom->tile_cols;
}

int lk_knn_build(const lk_knn_build_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_knn_build: null args");
    const lk_knn_build_args &a = *args;
    const lk_knn_geom &g = a.geom;
    LK_REQUIRE(a.d_ui_indptr && a.d_ui_cols && a.d_ui_vals && a.d_iu_indptr && a.d_iu_cols &&
                   a.d_iu_vals && a.d_tile_ptr && a.d_units && a.d_unit_ptr && a.d_sched && a.d_work_counter &&
                   a.d_status && a.d_part_cnt && a.d_tie_scratch,
               LK_ERR_INVALID, "lk_knn_build: null pointer");
    if (a.save_nbrs > 0)
        LK_REQUIRE(a.d_part_cols && a.d_part_vals, LK_ERR_INVALID, "truncated build needs partial lists");
    else
        LK_REQUIRE(a.d_pool_cols && a.d_pool_vals && a.d_pool_off && a.d_pool_cursor, LK_ERR_INVALID,
                   "unbounded build needs the pool");
    LK_REQUIRE(a.min_sim >= 0.0f, LK_ERR_INVALID, "min_sim must be non-negative");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (a.n_work == 0) return LK_OK;
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    const int smem = knn_smem_bytes(g);
    const unsigned grid = (unsigned)knn_grid(g, a.n_work);
    switch (g.warps) {
        case 8:
            LK_CUDA_TRY(cudaFuncSetAttribute(knn_build_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            knn_build_kernel<8><<<grid, 256, smem, st>>>(a);
            break;
        case 16:
            LK_CUDA_TRY(cudaFuncSetAttribute(knn_build_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            knn_build_kernel<16><<<grid, 512, smem, st>>>(a);
            break;
        case 32:
            LK_CUDA_TRY(cudaFuncSetAttribute(knn_build_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            knn_build_kernel<32><<<grid, 1024, smem, st>>>(a);
            break;
        default: set_error("unsupported warps per CTA %d", g.warps); return LK_ERR_INVALID;
    }
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_knn_merge_topk(const lk_knn_build_args *args, int32_t *d_out_cols, float *d_out_vals,
                      int32_t *d_out_cnt, void *stream)
{
    LK_REQUIRE(args && d_out_cols && d_out_vals && d_out_cnt, LK_ERR_INVALID, "lk_knn_merge_topk: null");
    const lk_knn_build_args &a = *args;
    LK_REQUIRE(a.save_nbrs > 0, LK_ERR_INVALID, "merge is for the truncated build");
    LK_REQUIRE(a.d_unit_ptr && a.max_units_per_item >= 1, LK_ERR_INVALID, "lk_knn_merge_topk: no unit table");
    const int cap = a.max_units_per_item * a.save_nbrs;
    const int smem = cap * 16;
    LK_REQUIRE(smem <= 200 * 1024, LK_ERR_UNSUPPORTED, "units per item * save_nbrs = %d too large to merge", cap);
    LK_CUDA_TRY(cudaFuncSetAttribute(knn_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int grid = std::min(a.geom.n_items, sm_count() * 16);
    if (grid < 1) grid = 1;
    knn_merge_kernel<<<grid, 128, smem, static_cast<cudaStream_t>(stream)>>>(a, d_out_cols, d_out_vals, d_out_cnt);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_knn_pool_to_csr(const lk_knn_build_args *args, const int64_t *d_out_indptr, int32_t *d_out_cols,
                       float *d_out_vals, void *stream)
{
    LK_REQUIRE(args && d_out_indptr && d_out_cols && d_out_vals, LK_ERR_INVALID, "lk_knn_pool_to_csr: null");
    pool_to_csr_kernel<<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, d_out_indptr,
                                                                                   d_out_cols, d_out_vals);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
