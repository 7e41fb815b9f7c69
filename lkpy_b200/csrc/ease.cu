// ease.cu — EASE scoring and fused top-n for sm_90a.
//
// Replaces EASEScorer.__call__ (knn/ease.py): `q_vec @ weights`, a dense f32 GEMV over the whole
// n_items x n_items weight matrix for a 0/1 query vector.  Only the rows of the query's history items matter, so
// the kernel streams exactly those rows: for query q with history H_q (deduplicated, ascending) and item j
//     s_j = +0.0f;  for h in H_q ascending: s_j = s_j + W[h, j]      (f32 adds, round to nearest)
// Every thread owns four adjacent columns of a column tile and keeps their sums in registers, so each sum sees
// the rows in history order by construction: no shared-memory accumulators, no atomics.  Rows are read with
// float4 loads when n_items is a multiple of 4 (every row start is then 16-byte aligned), and EASE_UNROLL rows'
// loads are issued before their adds so that enough bytes are in flight to stream from HBM.
//
// Score mode: one CTA per (query, column tile).  Rank mode: one CTA per query sweeping the tiles in ascending
// order; the EASE_CW compute threads write each tile's sums into one of two shared buffers and a separate heap
// warp offers the previous tile's buffer to argtopn's heap (topn_heap.cuh) while the next tile is summed, with
// the exact filter count < n || s > root (a full heap's root never decreases and a full heap rejects s <= root)
// and the query's exclusions skipped as argtopn skips NaN.
#include "common.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int EASE_CT = 256;             // compute threads per CTA
constexpr int EASE_TW = EASE_CT * 4;     // columns per tile
constexpr int EASE_UNROLL = 4;           // rows loaded ahead of their adds

// columns c .. c+3 of one row; columns at or beyond NI read as +0.0 (never stored)
template <bool VEC>
__device__ __forceinline__ float4 ease_load4(const float *__restrict__ row, const int c, const int NI)
{
    if constexpr (VEC) {
        if (c < NI) return __ldg(reinterpret_cast<const float4 *>(row + c));
        return make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
        float4 v;
        v.x = c < NI ? __ldg(row + c) : 0.f;
        v.y = c + 1 < NI ? __ldg(row + c + 1) : 0.f;
        v.z = c + 2 < NI ? __ldg(row + c + 2) : 0.f;
        v.w = c + 3 < NI ? __ldg(row + c + 3) : 0.f;
        return v;
    }
}

__device__ __forceinline__ void ease_add(float4 &s, const float4 v)
{
    s.x = __fadd_rn(s.x, v.x);
    s.y = __fadd_rn(s.y, v.y);
    s.z = __fadd_rn(s.z, v.z);
    s.w = __fadd_rn(s.w, v.w);
}

// the sums of columns c .. c+3 over the history rows hist[0 .. R-1], in that order
template <bool VEC>
__device__ __forceinline__ float4 ease_tile_sums(const float *__restrict__ W, const int32_t *__restrict__ hist,
                                                 const int R, const int c, const int NI)
{
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int t = 0;
    for (; t + EASE_UNROLL <= R; t += EASE_UNROLL) {
        float4 v[EASE_UNROLL];
#pragma unroll
        for (int u = 0; u < EASE_UNROLL; u++) v[u] = ease_load4<VEC>(W + (int64_t)__ldg(hist + t + u) * NI, c, NI);
#pragma unroll
        for (int u = 0; u < EASE_UNROLL; u++) ease_add(s, v[u]);
    }
    for (; t < R; t++) ease_add(s, ease_load4<VEC>(W + (int64_t)__ldg(hist + t) * NI, c, NI));
    return s;
}

template <bool RANK, bool VEC>
__global__ void __launch_bounds__(EASE_CT + (RANK ? 32 : 0)) ease_score_kernel(const lk_ease_score_args a)
{
    const int NI = a.n_items, T = (NI + EASE_TW - 1) / EASE_TW;
    const int tid = threadIdx.x;
    const int q = RANK ? (int)blockIdx.x : (int)(blockIdx.x / T);
    const int64_t h0 = a.d_hist_indptr[q];
    const int R = (int)(a.d_hist_indptr[q + 1] - h0);
    const int32_t *hist = a.d_hist_items + h0;
    const float qnan = __int_as_float(0x7fc00000);

    if constexpr (!RANK) {
        const int c = (int)(blockIdx.x % T) * EASE_TW + tid * 4;
        if (c >= NI) return;
        const float4 s = R == 0 ? make_float4(qnan, qnan, qnan, qnan) : ease_tile_sums<VEC>(a.d_w, hist, R, c, NI);
        float *out = a.d_scores + (int64_t)q * NI + c;
        if (VEC) {
            *reinterpret_cast<float4 *>(out) = s;
        } else {
            out[0] = s.x;
            if (c + 1 < NI) out[1] = s.y;
            if (c + 2 < NI) out[2] = s.z;
            if (c + 3 < NI) out[3] = s.w;
        }
    } else {
        __shared__ __align__(16) float buf[2][EASE_TW];
        __shared__ float s_hv[TOPN_MAX];
        __shared__ int32_t s_hk[TOPN_MAX];
        const int n = a.n;
        const int64_t o = (int64_t)q * n;
        if (R == 0) {  // no history: nothing is recommended
            for (int t = tid; t < n; t += blockDim.x) {
                a.d_out_idx[o + t] = -1;
                a.d_out_val[o + t] = qnan;
            }
            if (tid == 0) a.d_out_cnt[q] = 0;
            return;
        }
        const bool heap_warp = tid >= EASE_CT;
        const int lane = tid & 31;
        PairHeap<1> heap{s_hv, s_hk};
        int count = 0;  // heap warp: heap size and root, exclusion cursor
        float root = 0.0f;
        int64_t ec = 0, ee = 0;
        if (a.d_excl_indptr != nullptr) ec = a.d_excl_indptr[q], ee = a.d_excl_indptr[q + 1];

        // the heap warp offers tile k's sums from buf[k & 1] in ascending item order
        auto offer_tile = [&](const int k) {
            const float *b = buf[k & 1];
            for (int j0 = 0; j0 < EASE_TW; j0 += 32) {
                const int c = k * EASE_TW + j0 + lane;
                const float sc = b[j0 + lane];
                unsigned m = __ballot_sync(FULL, c < NI && !isnan(sc) && (count < n || sc > root));
                if (lane == 0) {
                    while (m) {
                        const int l = __ffs(m) - 1;
                        m &= m - 1u;
                        const int item = k * EASE_TW + j0 + l;
                        while (ec < ee && a.d_excl_items[ec] < item) ec++;
                        if (ec < ee && a.d_excl_items[ec] == item) continue;  // excluded: argtopn's NaN offer
                        topn_heap_offer(heap, count, root, n, PairHeap<1>::Ent{b[j0 + l], item});
                    }
                }
                count = __shfl_sync(FULL, count, 0);
                root = __shfl_sync(FULL, root, 0);
            }
        };

        for (int k = 0; k < T; k++) {
            if (!heap_warp) {
                const int c = k * EASE_TW + tid * 4;
                const float4 s = ease_tile_sums<VEC>(a.d_w, hist, R, c, NI);
                *reinterpret_cast<float4 *>(&buf[k & 1][tid * 4]) = s;
            } else if (k > 0) {
                offer_tile(k - 1);
            }
            // buf[k & 1] is complete, and the heap warp is done with buf[(k - 1) & 1]
            __syncthreads();
        }
        if (heap_warp) {
            offer_tile(T - 1);
            if (lane == 0) {
                topn_heap_sort(heap, count);
                for (int t = 0; t < n; t++) {
                    const bool in = t < count;
                    a.d_out_idx[o + t] = in ? heap.hk[t] : -1;
                    a.d_out_val[o + t] = in ? heap.hv[t] : qnan;
                }
                a.d_out_cnt[q] = count;
            }
        }
    }
}

template <bool RANK, bool VEC>
int launch_ease_score(const lk_ease_score_args &a, cudaStream_t st)
{
    const int64_t T = (a.n_items + EASE_TW - 1) / EASE_TW;
    const unsigned grid = RANK ? (unsigned)a.n_queries : (unsigned)(a.n_queries * T);
    ease_score_kernel<RANK, VEC><<<grid, EASE_CT + (RANK ? 32 : 0), 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_ease_score_batch(const lk_ease_score_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_ease_score_batch: null args");
    const lk_ease_score_args &a = *args;
    LK_REQUIRE(a.n_items >= 1, LK_ERR_INVALID, "lk_ease_score_batch: n_items must be positive");
    const int64_t T = (a.n_items + EASE_TW - 1) / EASE_TW;
    LK_REQUIRE(a.n_queries >= 0 && (int64_t)a.n_queries * T < 0x7fffffffLL, LK_ERR_UNSUPPORTED,
               "lk_ease_score_batch: n_queries * column tiles must be < 2^31");
    const bool rank = a.n != 0;
    if (rank)
        LK_REQUIRE(a.n >= 1 && a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED,
                   "lk_ease_score_batch: n must be 0 (score mode) or in 1..%d", TOPN_MAX);
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_w && a.d_hist_indptr && a.d_hist_items, LK_ERR_INVALID, "lk_ease_score_batch: null input");
    if (rank) {
        LK_REQUIRE(a.d_out_idx && a.d_out_val && a.d_out_cnt, LK_ERR_INVALID, "lk_ease_score_batch: null output");
        LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
                   "lk_ease_score_batch: d_excl_items is required with d_excl_indptr");
    } else {
        LK_REQUIRE(a.d_scores != nullptr, LK_ERR_INVALID, "lk_ease_score_batch: null score matrix");
    }
    // float4 rows need every row start 16-byte aligned: W itself and n_items % 4 == 0 (and the output likewise)
    const bool vec = a.n_items % 4 == 0 && reinterpret_cast<uintptr_t>(a.d_w) % 16 == 0 &&
                     (rank || reinterpret_cast<uintptr_t>(a.d_scores) % 16 == 0);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (rank) return vec ? launch_ease_score<true, true>(a, st) : launch_ease_score<true, false>(a, st);
    return vec ? launch_ease_score<false, true>(a, st) : launch_ease_score<false, false>(a, st);
}

}  // extern "C"
