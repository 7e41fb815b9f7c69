// basic.cu — the bias model and offset scoring for sm_90a: BiasModel.learn (src/lenskit/basic/bias.py:84-150) and the
// batched scoring and top-n of BiasScorer and PopScorer (basic/bias.py, basic/popularity.py).
//
// lk_bias_learn reproduces the host statements bit for bit (include/lkpy_b200.h):
//   * the global mean is np.mean of the f32 ratings: np.add.reduce starts from its identity +0.0 and adds
//     pairwise(r) in NumPy's order (pairwise.cuh), then divides in f64 by the count (an intp).  The
//     tree is cut at depth MEAN_DEPTH: one thread walks each subtree there (or a leaf reached above it), and one CTA
//     then combines the subtrees level by level, each node's value kept in the slot of its leftmost descendant;
//   * every entity's sum is np.add.at's: a chain of f64 adds in COO order, which no reordering may shorten.  A warp
//     owns an entity: its lanes load and centre the next 128 values while every lane runs the same chain over the
//     current ones, taking each value from its lane by shuffle.  The chain of the heaviest entity (81 k ratings for
//     the most rated item of ML-25M) is the floor of a pass; handing entities out longest first starts it at once,
//     and the rest of the pass runs beside it.
//
// lk_offset_score_batch scores s(q, i) = f32(f64(base[i]) + off[q]).  Rank mode is argtopn over every item in
// ascending order with topn_heap.cuh's heap, one thread per query as in topn.cu: adding the offset can merge
// neighbouring f32 values into ties (and popularity counts are mostly ties), so only the heap itself decides which
// tied items are kept and in what order.  All lanes of a warp read the same base[i] (one broadcast load), and after
// the first items nearly every score is rejected by one compare against the root.
#include <algorithm>

#include "common.cuh"
#include "pairwise.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int MEAN_DEPTH = 16;      // 2^16 subtrees of the mean's pairwise tree, walked in parallel
constexpr int MEAN_THREADS = 256;
constexpr int BIAS_THREADS = 256;   // 8 warps, one entity each at a time
constexpr int BIAS_CHUNKS = 4;      // 32-value chunks each lane holds: 128 values per step of the chain

// The mean's pairwise tree over r[0 .. nnz) is cut at MEAN_DEPTH (pairwise_node): a node at depth d with path p
// keeps its value in slot p << (MEAN_DEPTH - d).
__global__ void __launch_bounds__(MEAN_THREADS) mean_subtrees_kernel(const float *__restrict__ r, const int64_t nnz,
                                                                     float *__restrict__ part)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (1u << MEAN_DEPTH)) return;
    int64_t lo, n;
    if (!pairwise_node(nnz, MEAN_DEPTH, t, lo, n)) return;
    part[t] = pairwise_sum<F32Ops>([&](int64_t p) { return __ldg(r + p); }, lo, n);
}

// one CTA: the inner nodes above MEAN_DEPTH, deepest level first, then g = f32(f64(+0.0 + total) / nnz)
__global__ void __launch_bounds__(1024) mean_combine_kernel(const int64_t nnz, float *part, float *__restrict__ mean)
{
    if (nnz > 128) {
        for (int d = MEAN_DEPTH - 1; d >= 0; d--) {
            for (uint32_t p = threadIdx.x; p < (1u << d); p += blockDim.x) {
                int64_t lo, n;
                if (!pairwise_node(nnz, d, p, lo, n) || n <= 128) continue;  // absent, or a leaf: its slot is final
                const uint32_t s = p << (MEAN_DEPTH - d);
                part[s] = __fadd_rn(part[s], part[s + (1u << (MEAN_DEPTH - d - 1))]);
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        const float sum = __fadd_rn(0.0f, part[0]);
        *mean = __double2float_rn(__ddiv_rn((double)sum, (double)nnz));
    }
}

// one pass of BiasModel.learn: for every entity e, the f64 sum of its centred values vals[indptr[e] ..
// indptr[e+1]) in order, less sub[cols[p]] when sub is given, divided by the damped count and rounded to f32
template <bool F64C>
__global__ void __launch_bounds__(BIAS_THREADS)
bias_pass_kernel(const int32_t *__restrict__ order, const int n_ent, const int32_t *__restrict__ indptr,
                 const float *__restrict__ vals, const int32_t *__restrict__ cols, const float *__restrict__ sub,
                 const float *__restrict__ d_mean, const double damping, float *__restrict__ out)
{
    constexpr int STEP = 32 * BIAS_CHUNKS;
    const int lane = threadIdx.x & 31;
    const int warp = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    const int n_warps = (int)((gridDim.x * (unsigned)blockDim.x) >> 5);
    const float g = *d_mean;
    // an integral damping counts exactly: every partial count is an integer below 2^53
    const bool exact_count = damping == floor(damping) && damping < 4503599627370496.0;

    // the value np.add.at adds for rating p: c in its own type (ratings - g, then - ib[col]), widened to f64
    auto centred = [&](const int64_t p, const int64_t hi) -> double {
        if (p >= hi) return 0.0;
        const float rv = __ldg(vals + p);
        if constexpr (F64C) {
            double c = __dsub_rn((double)rv, (double)g);
            if (sub != nullptr) c = __dsub_rn(c, (double)__ldg(sub + __ldg(cols + p)));
            return c;
        } else {
            float c = __fsub_rn(rv, g);
            if (sub != nullptr) c = __fsub_rn(c, __ldg(sub + __ldg(cols + p)));
            return (double)c;
        }
    };

    for (int j = warp; j < n_ent; j += n_warps) {
        const int e = __ldg(order + j);
        const int64_t lo = __ldg(indptr + e), hi = __ldg(indptr + e + 1);
        double s = 0.0, cnt = damping;
        double v[BIAS_CHUNKS];
#pragma unroll
        for (int k = 0; k < BIAS_CHUNKS; k++) v[k] = centred(lo + k * 32 + lane, hi);
        for (int64_t base = lo; base < hi; base += STEP) {
            double nv[BIAS_CHUNKS];  // the next step's values, loaded while this step's chain runs
#pragma unroll
            for (int k = 0; k < BIAS_CHUNKS; k++) nv[k] = centred(base + STEP + k * 32 + lane, hi);
            const int m = (int)min(hi - base, (int64_t)STEP);  // warp-uniform
            if (m == STEP) {
#pragma unroll
                for (int k = 0; k < BIAS_CHUNKS; k++)
#pragma unroll
                    for (int t = 0; t < 32; t++) {
                        s = __dadd_rn(s, __shfl_sync(FULL, v[k], t));
                        if (!exact_count) cnt = __dadd_rn(cnt, 1.0);
                    }
            } else {
#pragma unroll
                for (int k = 0; k < BIAS_CHUNKS; k++)
                    for (int t = 0; t < 32; t++) {
                        const double x = __shfl_sync(FULL, v[k], t);
                        if (k * 32 + t < m) {
                            s = __dadd_rn(s, x);
                            if (!exact_count) cnt = __dadd_rn(cnt, 1.0);
                        }
                    }
            }
#pragma unroll
            for (int k = 0; k < BIAS_CHUNKS; k++) v[k] = nv[k];
        }
        if (exact_count) cnt = damping + (double)(hi - lo);
        // np.divide(sums, counts, out=f32, where=counts > 0): the f64 quotient rounded once; 0 where not written
        if (lane == 0) out[e] = cnt > 0.0 ? __double2float_rn(__ddiv_rn(s, cnt)) : 0.0f;
    }
}

template <bool F64C>
int launch_bias_pass(const int32_t *order, int n_ent, const int32_t *indptr, const float *vals, const int32_t *cols,
                     const float *sub, const float *mean, double damping, float *out, cudaStream_t st)
{
    if (n_ent == 0) return LK_OK;
    const int per_cta = BIAS_THREADS / 32;
    const int blocks = std::min((n_ent + per_cta - 1) / per_cta, sm_count() * (2048 / BIAS_THREADS));
    bias_pass_kernel<F64C><<<blocks, BIAS_THREADS, 0, st>>>(order, n_ent, indptr, vals, cols, sub, mean, damping,
                                                            out);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

__global__ void __launch_bounds__(256) offset_score_kernel(const lk_offset_score_args a)
{
    const int64_t total = (int64_t)a.n_queries * a.n_items;
    for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x) {
        const int64_t q = x / a.n_items;
        const int i = (int)(x - q * a.n_items);
        const double off = a.d_offset != nullptr ? __ldg(a.d_offset + q) : 0.0;
        a.d_scores[x] = __double2float_rn(__dadd_rn((double)__ldg(a.d_base + i), off));
    }
}

template <int NMAX>
__global__ void __launch_bounds__(128) offset_rank_kernel(const lk_offset_score_args a)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.n_queries) return;
    float hv[NMAX];
    int32_t hk[NMAX];
    PairHeap<1> h{hv, hk};  // the heap in the thread's own arrays (local memory)
    int count = 0;
    float root = 0.0f;
    const int n = a.n, NI = a.n_items;
    const double off = a.d_offset != nullptr ? a.d_offset[q] : 0.0;
    int64_t ec = 0, ee = 0;
    if (a.d_excl_indptr != nullptr) ec = a.d_excl_indptr[q], ee = a.d_excl_indptr[q + 1];

    auto offer = [&](const float b, const int32_t i) {
        const float s = __double2float_rn(__dadd_rn((double)b, off));
        if (s != s) return;                     // sorting.rs:142 accept = !is_nan
        if (count == n && !(s > root)) return;  // a full heap takes only a score above its root
        if (topn_excluded(a.d_excl_items, ec, ee, i)) return;
        topn_heap_offer(h, count, root, n, PairHeap<1>::Ent{s, i});
    };
    int i = 0;
    constexpr int UNR = 8;
    for (; i + UNR <= NI; i += UNR) {
        float b[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) b[u] = __ldg(a.d_base + i + u);
#pragma unroll
        for (int u = 0; u < UNR; u++) offer(b[u], i + u);
    }
    for (; i < NI; i++) offer(__ldg(a.d_base + i), i);

    topn_heap_sort(h, count);
    const int64_t o = (int64_t)q * n;
    for (int t = 0; t < n; t++) {
        a.d_out_idx[o + t] = t < count ? hk[t] : -1;
        a.d_out_val[o + t] = t < count ? hv[t] : __int_as_float(0x7fc00000);
    }
    a.d_out_cnt[q] = count;
}

}  // namespace lk

using namespace lk;

extern "C" {

int64_t lk_bias_learn_workspace_bytes(void) { return (int64_t)sizeof(float) << MEAN_DEPTH; }

int lk_bias_learn(const lk_bias_learn_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_bias_learn: null args");
    const lk_bias_learn_args &a = *args;
    LK_REQUIRE(a.nnz >= 1 && a.nnz < 0x7fffffffLL, LK_ERR_UNSUPPORTED, "lk_bias_learn: nnz must be in 1..2^31-1");
    LK_REQUIRE(a.n_users >= 0 && a.n_items >= 0, LK_ERR_INVALID, "lk_bias_learn: negative entity count");
    LK_REQUIRE(a.damping_user >= 0.0 && a.damping_item >= 0.0, LK_ERR_INVALID,
               "lk_bias_learn: damping must be non-negative");
    LK_REQUIRE(a.d_ratings && a.d_workspace && a.d_mean, LK_ERR_INVALID, "lk_bias_learn: null ratings or output");
    const bool items = a.d_item_bias != nullptr, users = a.d_user_bias != nullptr;
    if (items)
        LK_REQUIRE(a.d_item_indptr && a.d_item_ratings && a.d_item_order, LK_ERR_INVALID,
                   "lk_bias_learn: the item pass needs d_item_indptr, d_item_ratings and d_item_order");
    if (users)
        LK_REQUIRE(a.d_user_indptr && a.d_user_order && (!items || a.d_items), LK_ERR_INVALID,
                   "lk_bias_learn: the user pass needs d_user_indptr, d_user_order (and d_items after an item pass)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *part = static_cast<float *>(a.d_workspace);
    mean_subtrees_kernel<<<(1u << MEAN_DEPTH) / MEAN_THREADS, MEAN_THREADS, 0, st>>>(a.d_ratings, a.nnz, part);
    LK_CUDA_TRY(cudaGetLastError());
    mean_combine_kernel<<<1, 1024, 0, st>>>(a.nnz, part, a.d_mean);
    LK_CUDA_TRY(cudaGetLastError());
    auto pass = a.centered_f64 ? launch_bias_pass<true> : launch_bias_pass<false>;
    if (items) {
        const int rc = pass(a.d_item_order, a.n_items, a.d_item_indptr, a.d_item_ratings, nullptr, nullptr, a.d_mean,
                            a.damping_item, a.d_item_bias, st);
        if (rc != LK_OK) return rc;
    }
    if (users)
        return pass(a.d_user_order, a.n_users, a.d_user_indptr, a.d_ratings, a.d_items,
                    items ? a.d_item_bias : nullptr, a.d_mean, a.damping_user, a.d_user_bias, st);
    return LK_OK;
}

int lk_offset_score_batch(const lk_offset_score_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_offset_score_batch: null args");
    const lk_offset_score_args &a = *args;
    LK_REQUIRE(a.n_items >= 1 && a.n_queries >= 0, LK_ERR_INVALID, "lk_offset_score_batch: bad shape");
    const bool rank = a.n != 0;
    if (rank)
        LK_REQUIRE(a.n >= 1 && a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED,
                   "lk_offset_score_batch: n must be 0 (score mode) or in 1..%d", TOPN_MAX);
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_base != nullptr, LK_ERR_INVALID, "lk_offset_score_batch: null base scores");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!rank) {
        LK_REQUIRE(a.d_scores != nullptr, LK_ERR_INVALID, "lk_offset_score_batch: null score matrix");
        const int64_t total = (int64_t)a.n_queries * a.n_items;
        const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count() * 8);
        offset_score_kernel<<<blocks, 256, 0, st>>>(a);
        LK_CUDA_TRY(cudaGetLastError());
        return LK_OK;
    }
    LK_REQUIRE(a.d_out_idx && a.d_out_val && a.d_out_cnt, LK_ERR_INVALID, "lk_offset_score_batch: null output");
    LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
               "lk_offset_score_batch: d_excl_items is required with d_excl_indptr");
    const unsigned grid = (unsigned)((a.n_queries + 127) / 128);
    if (a.n <= 16)
        offset_rank_kernel<16><<<grid, 128, 0, st>>>(a);
    else if (a.n <= 128)
        offset_rank_kernel<128><<<grid, 128, 0, st>>>(a);
    else
        offset_rank_kernel<TOPN_MAX><<<grid, 128, 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
