// topn.cu — batched top-N selection for sm_90a.
//
// Replaces lenskit._accel.data.argtopn (src/accel/data/sorting.rs:131-170) — the
// step behind ItemList.top_n / TopNRanker (src/lenskit/data/_items.py:942-998,
// src/lenskit/basic/topn.py:32-69) — for a whole batch of score vectors at once.
//
// The reference selects with an indirect min-heap (src/accel/indirect/heap.rs):
// candidates are offered in index order, NaN is never accepted, a full heap takes
// a candidate only if it is strictly greater than the root, and the final order
// is a heap sort.  Which of several equal scores survive at the cut, and the
// order equal scores come out in, are consequences of the heap's element
// movement — so the kernel replays exactly that heap: one thread per score
// vector, candidates in index order, the same sift rules.
//
// That is affordable because of the layout: the batch is the *columns* of a
// row-major matrix scores[item][vector] (what Q · Xᵀ produces), so the 32 lanes of
// a warp read 32 consecutive floats per item — the scan is one coalesced pass over
// the matrix (HBM-bound: 4 bytes per score), and after the first few thousand
// items almost every candidate is rejected by a single compare against the root
// kept in a register.  Heap storage is per-thread local memory.

#include "common.cuh"
#include "topn_heap.cuh"

namespace lk {

template <int NMAX>
__global__ void __launch_bounds__(128)
topn_columns_kernel(const float *__restrict__ scores, const int64_t n_rows, const int64_t n_cols, const int64_t ld,
                    const int n, int32_t *__restrict__ out_idx, float *__restrict__ out_val,
                    int32_t *__restrict__ out_cnt)
{
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_cols) return;
    float hv[NMAX];
    int32_t hk[NMAX];
    PairHeap<1> h{hv, hk};  // the heap in the thread's own arrays (local memory)
    int count = 0;
    float root = 0.0f;  // hv[0] once the heap is full

    auto offer = [&](const float s, const int32_t i) {
        if (s != s) return;  // sorting.rs:142 accept = !is_nan
        topn_heap_offer(h, count, root, n, PairHeap<1>::Ent{s, i});
    };

    const float *col = scores + u;
    int64_t i = 0;
    constexpr int UNR = 8;  // independent loads in flight per thread
    for (; i + UNR <= n_rows; i += UNR) {
        float s[UNR];
#pragma unroll
        for (int q = 0; q < UNR; q++) s[q] = __ldcs(col + (i + q) * ld);
#pragma unroll
        for (int q = 0; q < UNR; q++) offer(s[q], (int32_t)(i + q));
    }
    for (; i < n_rows; i++) offer(__ldcs(col + i * ld), (int32_t)i);

    topn_heap_sort(h, count);  // heap.rs:56-65 topn_vec: descending score order
    for (int t = 0; t < n; t++) {
        out_idx[u * n + t] = t < count ? hk[t] : -1;
        if (out_val != nullptr) out_val[u * n + t] = t < count ? hv[t] : __int_as_float(0x7fc00000);
    }
    out_cnt[u] = count;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_topn_max(void) { return TOPN_MAX; }

int lk_topn_columns(const float *d_scores, int64_t n_rows, int64_t n_cols, int64_t ld, int32_t n, int32_t *d_out_idx,
                    float *d_out_val, int32_t *d_out_cnt, void *stream)
{
    LK_REQUIRE(n_rows >= 0 && n_cols >= 0 && ld >= n_cols, LK_ERR_INVALID, "lk_topn_columns: bad shape");
    LK_REQUIRE(n >= 1 && n <= TOPN_MAX, LK_ERR_UNSUPPORTED, "lk_topn_columns: n must be in 1..%d", TOPN_MAX);
    LK_REQUIRE(n_rows < (int64_t)INT32_MAX, LK_ERR_UNSUPPORTED, "lk_topn_columns: int32 item indices");
    if (n_cols == 0) return LK_OK;
    LK_REQUIRE(d_scores && d_out_idx && d_out_cnt, LK_ERR_INVALID, "lk_topn_columns: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((n_cols + 127) / 128);
    if (n <= 16)
        topn_columns_kernel<16><<<grid, 128, 0, st>>>(d_scores, n_rows, n_cols, ld, n, d_out_idx, d_out_val, d_out_cnt);
    else if (n <= 128)
        topn_columns_kernel<128><<<grid, 128, 0, st>>>(d_scores, n_rows, n_cols, ld, n, d_out_idx, d_out_val, d_out_cnt);
    else
        topn_columns_kernel<TOPN_MAX><<<grid, 128, 0, st>>>(d_scores, n_rows, n_cols, ld, n, d_out_idx, d_out_val,
                                                            d_out_cnt);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
