// als_recommend.cu — batched ALS scoring and top-n recommendation for sm_90a (lk_als_recommend_batch).
//
// The ALS scorers' batched inference: for query b with embedding x_b (ALSBase.embed_batch) and item i,
//     s = +0.0f;  for d = 0 .. k-1:  s = fmaf(Q[i,d], x_b[d], s)       one fp32 FMA chain, ascending d
//     s = s + item_offset[i];  s = s + query_offset[b]                 f32 adds, each only when given
// Score mode writes S[n_items][B] (what ALSBase.score_matrix returns).  Rank mode writes each query's
// argtopn over its candidates (every item ascending, minus the query's excluded items), ties included, and
// never stores the score matrix.  Both modes run the same dot-product code, so ranking a score-mode matrix
// with argtopn gives the rank-mode lists bit for bit.
//
// Arithmetic: SIMT FFMA, not tensor cores.  A register-blocked outer product over ascending d gives every output
// exactly the chain above, which the tests restate on the host (tests/als_oracle.py); mma.sync's
// accumulation order is not specified, and 3xTF32 does not give fp32 products.
//
// Tiling: a CTA of AR_THREADS threads owns AR_QT queries and keeps their X rows in shared memory (Xs[q][d]).
// It sweeps the item tiles (AR_IT items) in ascending order; Q is read through L2 (15 MB at the ML-25M shape,
// k = 64), AR_DK dimensions at a time, staged global -> registers -> shared memory one chunk ahead of the
// compute.  Each thread holds 8 items x 4 queries of accumulators: items ig + 16 j, queries 4 qg + jj.
// d beyond k is padded with +0 in Q and -0 in X: fmaf(+0, -0, s) = s + (-0) = s for every s, so the padding
// cannot change a bit (a +0 product would turn a -0 sum into +0).
//
// Rank mode's selection is the exact filter of knn_score.cu's ranking mode (DESIGN.md §4.7): after each item
// tile the survivors are the scores with count < n || s > root, root being the heap root as the previous tile
// left it (a full heap's root never decreases and a full heap rejects s <= root).  They are parked in shared
// memory with one mask bit each; then one thread per query takes its survivors in ascending item order, drops
// the excluded ones (argtopn returns on a NaN offer, and an excluded item is one) and offers the rest to its
// heap (topn_heap.cuh).  The heap lives in shared memory up to AR_HEAP_SMEM_N entries per query, beyond that in
// the caller's workspace.  There is no split of the item range: a split would need a heap merge that replays
// argtopn's tie order.
#include "common.cuh"
#include "topn_heap.cuh"

namespace lk {

constexpr int AR_THREADS = 256;
constexpr int AR_QT = 64;   // queries per CTA
constexpr int AR_IT = 128;  // items per tile
constexpr int AR_DK = 16;   // dimensions per staged chunk of Q
constexpr int AR_KMAX = 128;
constexpr int AR_QS = AR_DK + 4;  // Qs row stride (floats): float4 rows, conflict-free for the 8 lanes of a phase
constexpr int AR_SS = AR_QT + 1;  // Ss row stride
constexpr int AR_PRE = AR_IT * AR_DK / AR_THREADS;  // Q floats each thread stages per chunk
constexpr int AR_ROWS = AR_THREADS / AR_DK;         // items staged per pass of the CTA
constexpr int AR_HEAP_SMEM_N = 128;
static_assert(AR_THREADS == 16 * (AR_QT / 4) && AR_IT == 16 * 8, "16 x 16 threads of 8 items x 4 queries");
static_assert(AR_IT == 4 * 32, "four mask words per query and tile");

__host__ __device__ constexpr int ar_kpad(int k) { return (k + AR_DK - 1) / AR_DK * AR_DK; }
__host__ __device__ constexpr int ar_union_floats(bool rank) { return rank ? AR_IT * AR_SS : AR_IT * AR_QS; }

static size_t ar_smem_bytes(bool rank, int k, int n)
{
    size_t b = sizeof(float) * ((size_t)ar_union_floats(rank) + (size_t)AR_QT * (ar_kpad(k) + 4));
    if (rank) {
        // masks, counts, roots, exclusion cursors
        b += (sizeof(uint32_t) * 4 + sizeof(int32_t) + sizeof(float) + sizeof(int64_t)) * AR_QT;
        if (n <= AR_HEAP_SMEM_N) b += (sizeof(float) + sizeof(int32_t)) * (size_t)AR_QT * n;
    }
    return b;
}

template <bool RANK>
__global__ void __launch_bounds__(AR_THREADS, 2) als_recommend_kernel(const lk_als_rec_args a)
{
    extern __shared__ __align__(16) float ar_smem[];
    const int tid = threadIdx.x, ig = tid % 16, qg = tid / 16;
    const int k = a.k, KP = ar_kpad(k), XS = KP + 4, nc = KP / AR_DK;
    const int64_t NI = a.n_items;
    const int B = a.n_queries, n = a.n;
    const int q0 = blockIdx.x * AR_QT;
    const float *__restrict__ Q = a.d_items;
    float *U = ar_smem;  // Qs [AR_IT][AR_QS] while computing; rank mode: Ss [AR_IT][AR_SS] for the survivors
    float *Xs = U + ar_union_floats(RANK);
    uint32_t *mask = reinterpret_cast<uint32_t *>(Xs + AR_QT * XS);  // [4][AR_QT]
    int32_t *s_cnt = reinterpret_cast<int32_t *>(mask + 4 * AR_QT);
    float *s_root = reinterpret_cast<float *>(s_cnt + AR_QT);

    for (int e = tid; e < AR_QT * KP; e += AR_THREADS) {
        const int q = e / KP, d = e % KP, b = q0 + q;
        Xs[q * XS + d] = d < k ? (b < B ? a.d_queries[(int64_t)b * k + d] : 0.0f) : -0.0f;
    }
    // rank mode: thread tid < AR_QT selects for query q0 + tid.  Its heap size, root and exclusion cursor live in
    // shared memory between tiles (the filter reads the first two), which keeps them out of the GEMM's registers.
    const int my_b = q0 + tid;
    const bool selector = RANK && tid < AR_QT && my_b < B;
    int64_t *s_ec = reinterpret_cast<int64_t *>(s_root + AR_QT);
    auto my_heap = [&]() {  // one query's heap, interleaved with the CTA's others
        float *hv = n <= AR_HEAP_SMEM_N ? reinterpret_cast<float *>(s_ec + AR_QT)
                                        : reinterpret_cast<float *>(a.d_workspace) + (size_t)blockIdx.x * AR_QT * n * 2;
        return PairHeap<AR_QT>{hv + tid, reinterpret_cast<int32_t *>(hv + AR_QT * n) + tid};
    };
    if constexpr (RANK) {
        if (tid < AR_QT) {
#pragma unroll
            for (int w = 0; w < 4; w++) mask[w * AR_QT + tid] = 0u;
            s_cnt[tid] = 0;
            s_root[tid] = 0.0f;
            s_ec[tid] = selector && a.d_excl_indptr != nullptr ? a.d_excl_indptr[my_b] : 0;
        }
    }

    // staging of Q chunk g = (tile, chunk): element tid + AR_THREADS r is item tid / AR_DK + AR_ROWS r, dimension
    // tid % AR_DK
    const int64_t n_tiles = (NI + AR_IT - 1) / AR_IT;
    const int64_t G = n_tiles * nc;
    float pre[AR_PRE];
    auto load_chunk = [&](const int64_t g) {
        const int64_t i0 = (g / nc) * AR_IT;
        const int dd = (int)(g % nc) * AR_DK + tid % AR_DK;
#pragma unroll
        for (int r = 0; r < AR_PRE; r++) {
            const int64_t i = i0 + tid / AR_DK + AR_ROWS * r;
            pre[r] = i < NI && dd < k ? __ldg(Q + i * k + dd) : 0.0f;
        }
    };
    if (G > 0) load_chunk(0);

    for (int64_t tile = 0; tile < n_tiles; tile++) {
        float acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; j++)
#pragma unroll
            for (int jj = 0; jj < 4; jj++) acc[j][jj] = 0.0f;
        for (int c = 0; c < nc; c++) {
            __syncthreads();  // the previous chunk's readers (and the previous tile's selection) are done
#pragma unroll
            for (int r = 0; r < AR_PRE; r++) U[(tid / AR_DK + AR_ROWS * r) * AR_QS + tid % AR_DK] = pre[r];
            __syncthreads();
            if (tile * nc + c + 1 < G) load_chunk(tile * nc + c + 1);
            const float *qb = U + ig * AR_QS;
            const float *xb = Xs + 4 * qg * XS + c * AR_DK;
#pragma unroll
            for (int d = 0; d < AR_DK; d += 4) {
                float4 xv[4];
#pragma unroll
                for (int jj = 0; jj < 4; jj++) xv[jj] = *reinterpret_cast<const float4 *>(xb + jj * XS + d);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float4 qv = *reinterpret_cast<const float4 *>(qb + 16 * j * AR_QS + d);
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        float s = acc[j][jj];
                        s = __fmaf_rn(qv.x, xv[jj].x, s);
                        s = __fmaf_rn(qv.y, xv[jj].y, s);
                        s = __fmaf_rn(qv.z, xv[jj].z, s);
                        s = __fmaf_rn(qv.w, xv[jj].w, s);
                        acc[j][jj] = s;
                    }
                }
            }
        }
        const int64_t t0 = tile * AR_IT;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int64_t i = t0 + ig + 16 * j;
            const float ioff = a.d_item_offset != nullptr && i < NI ? a.d_item_offset[i] : 0.0f;
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                float s = acc[j][jj];
                if (a.d_item_offset != nullptr) s = __fadd_rn(s, ioff);
                const int b = q0 + 4 * qg + jj;
                if (a.d_query_offset != nullptr && b < B) s = __fadd_rn(s, a.d_query_offset[b]);
                acc[j][jj] = s;
            }
        }
        if constexpr (!RANK) {
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int64_t i = t0 + ig + 16 * j;
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    const int b = q0 + 4 * qg + jj;
                    if (i < NI && b < B) __stcs(a.d_scores + i * B + b, acc[j][jj]);
                }
            }
        } else {
            __syncthreads();  // Ss overlays Qs
            int cnt[4];
            float rt[4];
#pragma unroll
            for (int jj = 0; jj < 4; jj++) cnt[jj] = s_cnt[4 * qg + jj], rt[jj] = s_root[4 * qg + jj];
#pragma unroll
            for (int w = 0; w < 4; w++)  // mask word w holds items 32 w .. 32 w + 31: j = 2 w and 2 w + 1
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    uint32_t bits = 0u;
#pragma unroll
                    for (int j = 2 * w; j < 2 * w + 2; j++) {
                        const int il = ig + 16 * j;
                        const float s = acc[j][jj];
                        if (t0 + il < NI && q0 + 4 * qg + jj < B && s == s && (cnt[jj] < n || s > rt[jj])) {
                            U[il * AR_SS + 4 * qg + jj] = s;
                            bits |= 1u << (il % 32);
                        }
                    }
                    if (bits != 0u) atomicOr(&mask[w * AR_QT + 4 * qg + jj], bits);
                }
            __syncthreads();
            if (selector) {
                const int32_t *ex = a.d_excl_items;
                const int64_t ee = a.d_excl_indptr != nullptr ? a.d_excl_indptr[my_b + 1] : 0;
                int64_t ec = s_ec[tid];
                int count = s_cnt[tid];
                float root = s_root[tid];
                PairHeap<AR_QT> heap = my_heap();
#pragma unroll 1
                for (int w = 0; w < 4; w++) {
                    uint32_t m = mask[w * AR_QT + tid];
                    if (m == 0u) continue;
                    mask[w * AR_QT + tid] = 0u;
                    do {
                        const int il = w * 32 + __ffs(m) - 1;
                        m &= m - 1u;
                        const int32_t item = (int32_t)(t0 + il);
                        if (topn_excluded(ex, ec, ee, item)) continue;  // argtopn's NaN offer
                        topn_heap_offer(heap, count, root, n, PairHeap<AR_QT>::Ent{U[il * AR_SS + tid], item});
                    } while (m != 0u);
                }
                s_cnt[tid] = count;
                s_root[tid] = root;
                s_ec[tid] = ec;
            }
        }
    }

    if (selector) {
        const int count = s_cnt[tid];
        PairHeap<AR_QT> heap = my_heap();
        topn_heap_sort(heap, count);
        const int64_t o = (int64_t)my_b * n;
        for (int t = 0; t < n; t++) {
            const bool in = t < count;
            a.d_out_idx[o + t] = in ? heap.hk[t * AR_QT] : -1;
            a.d_out_val[o + t] = in ? heap.hv[t * AR_QT] : __int_as_float(0x7fc00000);
        }
        a.d_out_cnt[my_b] = count;
    }
}

template <bool RANK>
int launch_als_recommend(const lk_als_rec_args &a, cudaStream_t st)
{
    const size_t smem = ar_smem_bytes(RANK, a.k, a.n);
    LK_CUDA_TRY(cudaFuncSetAttribute(als_recommend_kernel<RANK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    LK_CUDA_TRY(cudaFuncSetAttribute(als_recommend_kernel<RANK>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    const unsigned grid = (unsigned)((a.n_queries + AR_QT - 1) / AR_QT);
    als_recommend_kernel<RANK><<<grid, AR_THREADS, smem, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // namespace lk

using namespace lk;

extern "C" {

int64_t lk_als_recommend_workspace_bytes(int32_t n_queries, int32_t n)
{
    if (n_queries <= 0 || n <= AR_HEAP_SMEM_N) return 0;
    const int64_t grid = ((int64_t)n_queries + AR_QT - 1) / AR_QT;
    return grid * AR_QT * n * (int64_t)(sizeof(float) + sizeof(int32_t));
}

int lk_als_recommend_batch(const lk_als_rec_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_als_recommend_batch: null args");
    const lk_als_rec_args &a = *args;
    LK_REQUIRE(a.k >= 1 && a.k <= AR_KMAX, LK_ERR_UNSUPPORTED, "lk_als_recommend_batch: k must be in 1..%d", AR_KMAX);
    LK_REQUIRE(a.n_items >= 0 && a.n_queries >= 0, LK_ERR_INVALID, "lk_als_recommend_batch: bad shape");
    LK_REQUIRE(a.n_items < (int64_t)INT32_MAX, LK_ERR_UNSUPPORTED, "lk_als_recommend_batch: int32 item numbers");
    const bool rank = a.n != 0;
    if (rank) {
        LK_REQUIRE(a.n >= 1 && a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED,
                   "lk_als_recommend_batch: n must be 0 (score mode) or in 1..%d", TOPN_MAX);
        LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
                   "lk_als_recommend_batch: d_excl_items is required with d_excl_indptr");
        LK_REQUIRE(lk_als_recommend_workspace_bytes(a.n_queries, a.n) == 0 || a.d_workspace != nullptr,
                   LK_ERR_INVALID, "lk_als_recommend_batch: n > %d needs the workspace", AR_HEAP_SMEM_N);
    }
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_queries != nullptr && (a.n_items == 0 || a.d_items != nullptr), LK_ERR_INVALID,
               "lk_als_recommend_batch: null factor pointer");
    if (rank) {
        LK_REQUIRE(a.d_out_idx && a.d_out_val && a.d_out_cnt, LK_ERR_INVALID, "lk_als_recommend_batch: null output");
    } else {
        if (a.n_items == 0) return LK_OK;
        LK_REQUIRE(a.d_scores != nullptr, LK_ERR_INVALID, "lk_als_recommend_batch: null score matrix");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return rank ? launch_als_recommend<true>(a, st) : launch_als_recommend<false>(a, st);
}

}  // extern "C"
