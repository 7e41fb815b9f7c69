// stochastic.cu — StochasticTopNRanker for sm_90a (src/lenskit/stochastic/_ranker.py:89-156): Plackett–Luce
// sampling by exponential keys over a batch of score rows, drawing NumPy's PCG64 stream.
//
// For each query the valid positions are those with a finite score that are not excluded; they are numbered in list
// order, and the k-th of them draws the k-th uniform of the query's stream.  Three launches:
//   1. prepare: one warp per row walks it in list order, 32 positions at a time, and takes the valid count and the
//      max and min of s = f32(score * scale).  Softmax and linear also compact s into the workspace (ballot prefix),
//      because NumPy sums the compacted values.
//   2. scan (one shared stream only): an exclusive scan of the counts gives each query's stream offset, continuing
//      from *d_position, which it advances by the batch's draws.
//   3. keys: one warp per row.  The normaliser (softmax, linear) is +0.0 + pairwise(w) in NumPy's order: the tree is
//      cut into 32 subtrees (pairwise_node), each lane walks one, and the lanes combine them level by level as
//      basic.cu's mean does.  Then the row is walked again: lane l, the r-th valid position of its chunk, takes the
//      state M^(r+1) S + G_(r+1) inc from the chunk's start state S, outputs XSL-RR of it, and the chunk advances S
//      by its valid count.  key = log(u) / f64(max(w, FLT_MIN)).  Rank mode offers the keys that beat the heap root
//      to a per-warp heap in shared memory (topn_heap.cuh with f64 keys), one lane in list order, so ties are cut
//      and ordered as argtopn does; key mode writes every key.
// Every f32 step of the reference is an explicit _rn intrinsic; exp is (float)exp((double)x), log the f64 log.
#include <algorithm>
#include <cfloat>
#include <climits>

#include "common.cuh"
#include "pairwise.cuh"
#include "topn_heap.cuh"

namespace lk {

using u128 = unsigned __int128;

constexpr int ST_WARPS = 8;                                     // warps (queries) per CTA
constexpr int ST_LANE_JUMPS = 33;                               // (M^j, G_j), j = 0..32
constexpr int ST_POW_JUMPS = 64;                                // (M^(2^t), G_(2^t)), t = 0..63
constexpr int ST_SUM_DEPTH = 5;                                 // 32 subtrees of the normaliser's tree
constexpr int ST_MAX_ITEMS = INT_MAX - 64;                      // positions are int32, chunk ends included

struct Jump {
    u128 mul, add;  // s -> mul * s + add * inc
};

__device__ __forceinline__ Jump load_jump(const uint64_t *w)
{
    return {((u128)w[0] << 64) | w[1], ((u128)w[2] << 64) | w[3]};
}

__device__ __forceinline__ u128 apply(const Jump &j, const u128 s, const u128 inc) { return j.mul * s + j.add * inc; }

// PCG64's output function (XSL-RR) of a state
__device__ __forceinline__ uint64_t xsl_rr(const u128 s)
{
    const uint64_t hi = (uint64_t)(s >> 64), x = hi ^ (uint64_t)s;
    const unsigned rot = (unsigned)(hi >> 58);
    return (x >> rot) | (x << ((64u - rot) & 63u));
}

// the exclusion bits of positions [base, base + 32) from the query's ascending exclusions ex[ec .. ee), advancing
// the cursor past them; every lane returns the same mask
__device__ __forceinline__ uint32_t chunk_excluded(const int32_t *ex, int64_t &ec, const int64_t ee, const int base,
                                                   const int lane)
{
    uint32_t bits = 0;
    for (;;) {
        const int64_t i = ec + lane;
        const int e = i < ee ? __ldg(ex + i) : INT_MAX;
        const bool below = e < base + 32;
        bits |= __reduce_or_sync(FULL, below && e >= base ? 1u << (e - base) : 0u);
        const int k = __popc(__ballot_sync(FULL, below));
        ec += k;
        if (k < 32) return bits;
    }
}

// one row's walk in list order: calls f(base, valid mask, ok, position, s = f32(score * scale)) once per chunk of 32
template <typename F>
__device__ __forceinline__ void walk_row(const lk_stochastic_args &a, const int q, const int lane, F &&f)
{
    const float *row = a.d_scores + (int64_t)q * a.row_stride;
    int64_t ec = 0, ee = 0;
    if (a.d_excl_indptr != nullptr) ec = __ldg(a.d_excl_indptr + q), ee = __ldg(a.d_excl_indptr + q + 1);
    for (int base = 0; base < a.n_items; base += 32) {
        const uint32_t ex = chunk_excluded(a.d_excl_items, ec, ee, base, lane);
        const int i = base + lane;
        float s = 0.0f;
        bool ok = false;
        if (i < a.n_items) {
            const float x = __ldg(row + (int64_t)i * a.item_stride);
            ok = isfinite(x) && !((ex >> lane) & 1u);  // np.isfinite: NaN and ±inf are both dropped
            s = __fmul_rn(x, a.scale);
        }
        f(base, __ballot_sync(FULL, ok), ok, i, s);
    }
}

struct StWork {
    int32_t *cnt;
    float *mx, *mn;
    int64_t *off;
    float *compact;  // [B][n_items], or null
};

__host__ __device__ inline StWork st_work(void *ws, const int64_t B, const bool compact)
{
    char *p = static_cast<char *>(ws);
    const int64_t b8 = (B + 1) / 2 * 2;  // keeps the int64 offsets 8-byte aligned
    StWork w;
    w.cnt = reinterpret_cast<int32_t *>(p);
    w.mx = reinterpret_cast<float *>(p + 4 * b8);
    w.mn = reinterpret_cast<float *>(p + 8 * b8);
    w.off = reinterpret_cast<int64_t *>(p + 12 * b8);
    w.compact = compact ? reinterpret_cast<float *>(p + 20 * b8) : nullptr;
    return w;
}

__host__ __device__ inline int64_t st_work_bytes(const int64_t B, const int64_t L, const bool compact)
{
    const int64_t b8 = (B + 1) / 2 * 2;
    return 20 * b8 + (compact ? 4 * B * L : 0);
}

__device__ __forceinline__ uint32_t lanemask_lt(const int lane) { return (1u << lane) - 1u; }

__global__ void __launch_bounds__(ST_WARPS * 32) stoch_prepare_kernel(const lk_stochastic_args a, const StWork w)
{
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
    if (q >= a.n_queries) return;  // warp-uniform
    float *out = w.compact != nullptr ? w.compact + (int64_t)q * a.n_items : nullptr;
    int c = 0;
    float hi = -INFINITY, lo = INFINITY;
    walk_row(a, q, lane, [&](int, const uint32_t vm, const bool ok, int, const float s) {
        if (ok) {
            hi = fmaxf(hi, s), lo = fminf(lo, s);
            if (out != nullptr) out[c + __popc(vm & lanemask_lt(lane))] = s;
        }
        c += __popc(vm);
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, o));
        lo = fminf(lo, __shfl_xor_sync(FULL, lo, o));
    }
    if (lane == 0) w.cnt[q] = c, w.mx[q] = hi, w.mn[q] = lo;
}

// one CTA: off[q] = *pos + sum(cnt[0 .. q)), then *pos += sum(cnt)
__global__ void __launch_bounds__(1024) stoch_scan_kernel(const StWork w, const int B, int64_t *pos)
{
    __shared__ int64_t tot[32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int per = (B + 1023) / 1024, lo = min(B, t * per), hi = min(B, lo + per);
    const int64_t base = *pos;
    int64_t s = 0;
    for (int i = lo; i < hi; i++) s += w.cnt[i];
    int64_t v = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t u = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) tot[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int64_t x = tot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t u = __shfl_up_sync(FULL, x, o);
            if (lane >= o) x += u;
        }
        tot[lane] = x;
    }
    __syncthreads();
    int64_t e = base + (warp > 0 ? tot[warp - 1] : 0) + v - s;
    for (int i = lo; i < hi; i++) w.off[i] = e, e += w.cnt[i];
    if (t == 0) *pos = base + tot[31];  // every thread read *pos before the first barrier
}

// a heap of (f64 key, int32 position) in shared memory
struct KeyHeap {
    struct Ent {
        double v;
        int32_t k;
    };
    double *hv;
    int32_t *hk;
    __device__ __forceinline__ double val(const int p) const { return hv[p]; }
    __device__ __forceinline__ Ent get(const int p) const { return {hv[p], hk[p]}; }
    __device__ __forceinline__ void put(const int p, const Ent e) { hv[p] = e.v, hk[p] = e.k; }
};

template <bool RANK>
__global__ void __launch_bounds__(ST_WARPS * 32) stoch_key_kernel(const lk_stochastic_args a, const StWork w)
{
    __shared__ Jump lane_jump[ST_LANE_JUMPS];
    extern __shared__ __align__(16) unsigned char st_smem[];
    for (int j = threadIdx.x; j < ST_LANE_JUMPS; j += blockDim.x) lane_jump[j] = load_jump(a.d_jump + 4 * j);
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int q = blockIdx.x * ST_WARPS + wid;
    if (q >= a.n_queries) return;  // warp-uniform, after the only barrier
    const int N = w.cnt[q];
    const float *row = a.d_scores + (int64_t)q * a.row_stride;

    if (N == 0) {  // nothing valid: nothing is drawn
        if constexpr (RANK) {
            for (int t = lane; t < a.n; t += 32) {
                a.d_out_idx[(int64_t)q * a.n + t] = -1;
                a.d_out_val[(int64_t)q * a.n + t] = __int_as_float(0x7fc00000);
                if (a.d_out_key != nullptr) a.d_out_key[(int64_t)q * a.n + t] = __longlong_as_double(0x7ff8000000000000LL);
            }
        } else {
            for (int i = lane; i < a.n_items; i += 32)
                a.d_keys[(int64_t)q * a.n_items + i] = __longlong_as_double(0x7ff8000000000000LL);
        }
        if (lane == 0) a.d_out_cnt[q] = 0;
        return;
    }

    // the normaliser: +0.0 + pairwise(t(s)) over the compacted values, 32 subtrees then NumPy's tree above them
    const float mx = w.mx[q], mn = w.mn[q];
    const int tf = a.transform;
    float tot = 0.0f, rf = 0.0f;
    bool uniform = false;
    if (tf == LK_STOCH_LINEAR) {
        const double r = __dsub_rn((double)mx, (double)mn);
        uniform = !(r > 0.0);
        rf = __double2float_rn(r);
    }
    if (tf == LK_STOCH_SOFTMAX || (tf == LK_STOCH_LINEAR && !uniform)) {
        const float *cs = w.compact + (int64_t)q * a.n_items;
        auto term = [&](const int64_t p) {
            const float s = cs[p];
            return tf == LK_STOCH_SOFTMAX ? __double2float_rn(exp((double)__fsub_rn(s, mx)))
                                          : __fdiv_rn(__fsub_rn(s, mn), rf);
        };
        int64_t lo, n;
        float v = 0.0f;
        if (pairwise_node(N, ST_SUM_DEPTH, lane, lo, n)) v = pairwise_sum<F32Ops>(term, lo, n);
        if (N > 128) {
            for (int d = ST_SUM_DEPTH - 1; d >= 0; d--) {
                const int span = 1 << (ST_SUM_DEPTH - d);
                const float right = __shfl_down_sync(FULL, v, span / 2);
                if ((lane & (span - 1)) == 0 && pairwise_node(N, d, lane >> (ST_SUM_DEPTH - d), lo, n) && n > 128)
                    v = __fadd_rn(v, right);
            }
        }
        tot = __fadd_rn(0.0f, __shfl_sync(FULL, v, 0));
        if (tf == LK_STOCH_LINEAR) uniform = !(tot > 0.0f);
    }
    const float uw = __fdiv_rn(1.0f, __int2float_rn(N));
    auto weight = [&](const float s) -> float {
        if (tf == LK_STOCH_SOFTMAX) return __fdiv_rn(__double2float_rn(exp((double)__fsub_rn(s, mx))), tot);
        if (tf == LK_STOCH_LINEAR) return uniform ? uw : __fdiv_rn(__fdiv_rn(__fsub_rn(s, mn), rf), tot);
        return s;
    };

    // the stream: the query's own state, or the shared one advanced by the query's offset
    const uint64_t *sw = a.d_state + (a.shared_stream ? 0 : 4 * (int64_t)q);
    u128 S = ((u128)sw[0] << 64) | sw[1];
    const u128 inc = ((u128)sw[2] << 64) | sw[3];
    if (a.shared_stream) {
        const uint64_t off = (uint64_t)w.off[q];
        for (int t = 0; t < ST_POW_JUMPS; t++)
            if ((off >> t) & 1u) S = apply(load_jump(a.d_jump + 4 * (ST_LANE_JUMPS + t)), S, inc);
    }

    KeyHeap h{reinterpret_cast<double *>(st_smem) + (int64_t)wid * a.n,
              reinterpret_cast<int32_t *>(st_smem + (size_t)ST_WARPS * a.n * sizeof(double)) + (int64_t)wid * a.n};
    int count = 0;
    double root = 0.0;
    walk_row(a, q, lane, [&](const int base, const uint32_t vm, const bool ok, const int i, const float s) {
        double key = __longlong_as_double(0x7ff8000000000000LL);
        if (ok) {
            const u128 st = apply(lane_jump[__popc(vm & lanemask_lt(lane)) + 1], S, inc);
            const double u = (double)(xsl_rr(st) >> 11) * 0x1.0p-53;  // uniform(0, 1): next_double
            const float wt = weight(s);
            const float wc = wt < FLT_MIN ? FLT_MIN : wt;              // np.maximum(w, smallest normal)
            key = __ddiv_rn(log(u), (double)wc);
        }
        S = apply(lane_jump[__popc(vm)], S, inc);
        if constexpr (RANK) {
            uint32_t cm = __ballot_sync(FULL, ok && key == key && (count < a.n || key > root));
            while (cm != 0u) {
                const int l = __ffs(cm) - 1;
                cm &= cm - 1u;
                const double k = __shfl_sync(FULL, key, l);
                if (lane == 0) topn_heap_offer(h, count, root, a.n, KeyHeap::Ent{k, base + l});
            }
            count = __shfl_sync(FULL, count, 0);
            root = __shfl_sync(FULL, root, 0);
        } else {
            if (i < a.n_items) a.d_keys[(int64_t)q * a.n_items + i] = key;
        }
    });
    if constexpr (RANK) {
        if (lane == 0) topn_heap_sort(h, count);
        __syncwarp();
        const int64_t o = (int64_t)q * a.n;
        for (int t = lane; t < a.n; t += 32) {
            const bool has = t < count;
            const int p = has ? h.hk[t] : -1;
            a.d_out_idx[o + t] = p;
            a.d_out_val[o + t] = has ? __ldg(row + (int64_t)p * a.item_stride) : __int_as_float(0x7fc00000);
            if (a.d_out_key != nullptr) a.d_out_key[o + t] = has ? h.hv[t] : __longlong_as_double(0x7ff8000000000000LL);
        }
        if (lane == 0) a.d_out_cnt[q] = count;
    } else if (lane == 0) {
        a.d_out_cnt[q] = N;
    }
}

}  // namespace lk

using namespace lk;

extern "C" {

int64_t lk_stochastic_workspace_bytes(int64_t n_queries, int64_t n_items, int32_t transform)
{
    if (n_queries < 0 || n_items < 0) return -1;
    return st_work_bytes(n_queries, n_items, transform == LK_STOCH_SOFTMAX || transform == LK_STOCH_LINEAR);
}

int lk_stochastic_topn(const lk_stochastic_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_stochastic_topn: null args");
    const lk_stochastic_args &a = *args;
    LK_REQUIRE(a.n_queries >= 0 && a.n_items >= 0, LK_ERR_INVALID, "lk_stochastic_topn: negative shape");
    LK_REQUIRE(a.n_items <= ST_MAX_ITEMS, LK_ERR_UNSUPPORTED, "lk_stochastic_topn: positions must fit in int32");
    LK_REQUIRE(a.n >= 0, LK_ERR_INVALID, "lk_stochastic_topn: negative n");
    LK_REQUIRE(a.n <= TOPN_MAX, LK_ERR_UNSUPPORTED,
               "lk_stochastic_topn: n must be 0 (key mode) or in 1..%d", TOPN_MAX);
    LK_REQUIRE(a.transform == LK_STOCH_NONE || a.transform == LK_STOCH_SOFTMAX || a.transform == LK_STOCH_LINEAR,
               LK_ERR_INVALID, "lk_stochastic_topn: unknown transform %d", a.transform);
    if (a.n_queries == 0) return LK_OK;
    LK_REQUIRE(a.d_scores && a.d_state && a.d_jump && a.d_workspace && a.d_out_cnt, LK_ERR_INVALID,
               "lk_stochastic_topn: null scores, state, jump table, workspace or counts");
    LK_REQUIRE(!a.shared_stream || a.d_position, LK_ERR_INVALID, "lk_stochastic_topn: a shared stream needs d_position");
    LK_REQUIRE(a.d_excl_indptr == nullptr || a.d_excl_items != nullptr, LK_ERR_INVALID,
               "lk_stochastic_topn: d_excl_items is required with d_excl_indptr");
    const bool rank = a.n > 0;
    if (rank)
        LK_REQUIRE(a.d_out_idx && a.d_out_val, LK_ERR_INVALID, "lk_stochastic_topn: null rank outputs");
    else
        LK_REQUIRE(a.d_keys != nullptr, LK_ERR_INVALID, "lk_stochastic_topn: null key matrix");
    const int64_t need = lk_stochastic_workspace_bytes(a.n_queries, a.n_items, a.transform);
    LK_REQUIRE(a.workspace_bytes >= need, LK_ERR_INVALID, "lk_stochastic_topn: workspace of %lld bytes, %lld needed",
               (long long)a.workspace_bytes, (long long)need);

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool compact = a.transform != LK_STOCH_NONE;
    const StWork w = st_work(a.d_workspace, a.n_queries, compact);
    const unsigned grid = (unsigned)((a.n_queries + ST_WARPS - 1) / ST_WARPS);
    stoch_prepare_kernel<<<grid, ST_WARPS * 32, 0, st>>>(a, w);
    LK_CUDA_TRY(cudaGetLastError());
    if (a.shared_stream) {
        stoch_scan_kernel<<<1, 1024, 0, st>>>(w, a.n_queries, a.d_position);
        LK_CUDA_TRY(cudaGetLastError());
    }
    if (rank) {
        const size_t smem = (size_t)ST_WARPS * a.n * (sizeof(double) + sizeof(int32_t));
        LK_CUDA_TRY(cudaFuncSetAttribute(stoch_key_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        stoch_key_kernel<true><<<grid, ST_WARPS * 32, smem, st>>>(a, w);
    } else {
        stoch_key_kernel<false><<<grid, ST_WARPS * 32, 0, st>>>(a, w);
    }
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
