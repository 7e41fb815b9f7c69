// fair.cu — FAIRReranker for sm_90a (src/lenskit/reranking/fair.py): the FA*IR merge of ranked lists, batched,
// and fused after argtopn's top-N selection from a score matrix.
//
// The merge reads only positions and protected flags.  With P the protected positions and U the others, both in list
// order, step i takes the head of P while the protected count is below m[i], else the earlier of the two heads.  One
// warp per list: the heads are warp-uniform, and the next head of a queue is found 32 flags at a time by a ballot, so
// a list of L positions costs L / 32 ballots per queue plus one per step.
//
// The score mode selects each row's top N as topn.cu does (candidates offered in item order to argtopn's heap,
// topn_heap.cuh, here in shared memory with lane 0 offering what beats the root; an excluded item is a NaN offer),
// heap-sorts it, and merges that N-list in the same kernel.  The whole N-heap is needed: which of several equal
// scores survive the cut, and the order they come out in, follow the heap's arrangement, and the merge's choice
// between a protected and an unprotected head depends on that order.
#include <climits>

#include "common.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int FAIR_WARPS = 8;  // warps (lists or queries) per CTA

// the first position in [x, L) whose flag is `want`, or L; every lane returns the same position
template <class F>
__device__ __forceinline__ int fair_next(const F &flag, const int x, const int L, const bool want, const int lane)
{
    for (int base = x; base < L; base += 32) {
        const int p = base + lane;
        const unsigned b = __ballot_sync(FULL, p < L && flag(p) == want);
        if (b != 0u) return base + __ffs(b) - 1;
    }
    return L;
}

// fair.py __call__'s loop over a list of L positions to length len (<= L): emit(i, position) on lane 0 for each step
template <class F, class E>
__device__ __forceinline__ void fair_merge(const F &flag, const int L, const int len, const int32_t *m, const int lane,
                                           const E &emit)
{
    int pp = fair_next(flag, 0, L, true, lane), pu = fair_next(flag, 0, L, false, lane), prot = 0;
    for (int i = 0; i < len; i++) {
        // the protected head when the constraint asks for it, when U is empty, or when it comes first
        if (pp < L && (prot < __ldg(m + i) || pu >= L || pp < pu)) {
            if (lane == 0) emit(i, pp);
            prot++;
            pp = fair_next(flag, pp + 1, L, true, lane);
        } else {
            if (lane == 0) emit(i, pu);
            pu = fair_next(flag, pu + 1, L, false, lane);
        }
    }
}

__global__ void __launch_bounds__(FAIR_WARPS * 32) fair_lists_kernel(const lk_fair_args a)
{
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * FAIR_WARPS + (threadIdx.x >> 5);
    if (q >= a.n_queries) return;  // warp-uniform
    const int64_t o = __ldg(a.d_list_indptr + q);
    const int L = (int)(__ldg(a.d_list_indptr + q + 1) - o);
    const int len = min(min(__ldg(a.d_list_len + q), a.n), L);
    const uint8_t *f = a.d_list_protected + o;
    int32_t *out = a.d_out_idx + (int64_t)q * a.n;
    fair_merge([&](const int p) { return __ldg(f + p) != 0; }, L, len, a.d_m, lane,
               [&](const int i, const int p) { out[i] = p; });
    for (int t = len + lane; t < a.n; t += 32) out[t] = -1;
    if (lane == 0) a.d_out_cnt[q] = len;
}

__global__ void __launch_bounds__(FAIR_WARPS * 32) fair_scores_kernel(const lk_fair_args a)
{
    extern __shared__ __align__(16) unsigned char fair_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int q = blockIdx.x * FAIR_WARPS + wid;
    if (q >= a.n_queries) return;  // warp-uniform; the kernel has no barrier
    const int N = a.n_candidates;
    PairHeap<1> h{reinterpret_cast<float *>(fair_smem) + (int64_t)wid * N,
                  reinterpret_cast<int32_t *>(fair_smem + (size_t)FAIR_WARPS * N * sizeof(float)) + (int64_t)wid * N};
    const float *row = a.d_scores + (int64_t)q * a.row_stride;
    int64_t ec = 0, ee = 0;  // lane 0's exclusion cursor
    if (a.d_excl_indptr != nullptr) ec = __ldg(a.d_excl_indptr + q), ee = __ldg(a.d_excl_indptr + q + 1);
    int count = 0;
    float root = 0.0f;
    for (int base = 0; base < a.n_items; base += 32) {
        const int i = base + lane;
        const float s = i < a.n_items ? __ldg(row + (int64_t)i * a.item_stride) : __int_as_float(0x7fc00000);
        // an offer that does not beat the root of a full heap is rejected whatever comes before it in the chunk
        uint32_t cm = __ballot_sync(FULL, s == s && (count < N || s > root));
        while (cm != 0u) {
            const int l = __ffs(cm) - 1;
            cm &= cm - 1u;
            const float v = __shfl_sync(FULL, s, l);
            if (lane == 0 && !topn_excluded(a.d_excl_items, ec, ee, base + l))
                topn_heap_offer(h, count, root, N, PairHeap<1>::Ent{v, base + l});
        }
        count = __shfl_sync(FULL, count, 0);
        root = __shfl_sync(FULL, root, 0);
    }
    if (lane == 0) topn_heap_sort(h, count);
    __syncwarp();

    // the merge over the sorted candidates: position p is the item h.hk[p] with the score h.hv[p]
    const int len = min(a.n, count);
    const int64_t o = (int64_t)q * a.n;
    fair_merge([&](const int p) { return __ldg(a.d_item_protected + h.hk[p]) != 0; }, count, len, a.d_m, lane,
               [&](const int i, const int p) {
                   a.d_out_idx[o + i] = h.hk[p];
                   if (a.d_out_val != nullptr) a.d_out_val[o + i] = h.hv[p];
               });
    for (int t = len + lane; t < a.n; t += 32) {
        a.d_out_idx[o + t] = -1;
        if (a.d_out_val != nullptr) a.d_out_val[o + t] = __int_as_float(0x7fc00000);
    }
    if (lane == 0) a.d_out_cnt[q] = len;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_fair_rerank(const lk_fair_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_fair_rerank: null args");
    const lk_fair_args &a = *args;
    LK_REQUIRE(a.mode == LK_FAIR_LISTS || a.mode == LK_FAIR_SCORES, LK_ERR_INVALID, "lk_fair_rerank: unknown mode %d",
               a.mode);
    LK_REQUIRE(a.n_queries >= 0, LK_ERR_INVALID, "lk_fair_rerank: negative batch");
    LK_REQUIRE(a.n >= 1, LK_ERR_INVALID, "lk_fair_rerank: n must be positive");
    LK_REQUIRE(a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED, "lk_fair_rerank: n must be in 1..%d", TOPN_MAX);
    const bool scores = a.mode == LK_FAIR_SCORES;
    if (scores) {
        LK_REQUIRE(a.n_candidates >= 1, LK_ERR_INVALID, "lk_fair_rerank: n_candidates must be positive");
        LK_REQUIRE(a.n_candidates <= TOPN_MAX, LK_ERR_UNSUPPORTED, "lk_fair_rerank: n_candidates must be in 1..%d",
                   TOPN_MAX);
        LK_REQUIRE(a.n_items >= 0, LK_ERR_INVALID, "lk_fair_rerank: negative n_items");
        LK_REQUIRE(a.n_items <= INT_MAX - 32, LK_ERR_UNSUPPORTED, "lk_fair_rerank: item numbers must fit in int32");
    }
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_m && a.d_out_idx && a.d_out_cnt, LK_ERR_INVALID, "lk_fair_rerank: null m, outputs or counts");
    if (scores) {
        LK_REQUIRE(a.d_scores && a.d_item_protected, LK_ERR_INVALID, "lk_fair_rerank: null scores or item flags");
        LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
                   "lk_fair_rerank: d_excl_items is required with d_excl_indptr");
    } else {
        LK_REQUIRE(a.d_list_indptr && a.d_list_protected && a.d_list_len, LK_ERR_INVALID,
                   "lk_fair_rerank: null list offsets, flags or lengths");
    }

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((a.n_queries + FAIR_WARPS - 1) / FAIR_WARPS);
    if (scores) {
        const size_t smem = (size_t)FAIR_WARPS * a.n_candidates * (sizeof(float) + sizeof(int32_t));
        LK_CUDA_TRY(cudaFuncSetAttribute(fair_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        fair_scores_kernel<<<grid, FAIR_WARPS * 32, smem, st>>>(a);
    } else {
        fair_lists_kernel<<<grid, FAIR_WARPS * 32, 0, st>>>(a);
    }
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
