// knn_score.cu — batched item-kNN neighbourhood scoring for sm_90a.
//
// Replaces src/accel/knn/item_score.rs:22-111 (score_explicit / score_implicit)
// and the ScoreAccumulator of src/accel/knn/accum.rs:16-239, batched over many
// queries (the reference scores one query per call, single-threaded).
//
// Semantics kept exactly (DESIGN.md §kNN-score):
//   * reference items are visited in history order, each one's similarity row
//     in column order; a target's accumulator takes the first `max_nbrs`
//     contributions as a vector (accum.rs:86-98) whose sums are taken in push
//     order — reproduced here by running sums updated in the same order;
//   * a target that receives more than `max_nbrs` contributions switches to a
//     min-heap (accum.rs:73-82,100-117).  Those targets are re-scored by a
//     per-lane emulation of the Rust std BinaryHeap element movement so that
//     the survivor set under ties and the summation order match;
//   * null (negative) reference items are skipped, null targets give NaN / -1.
//
// One warp owns one query: lanes spread over the entries of a similarity row,
// history entries are processed one after the other (order is the contract).
// A per-warp `slotmap` (n_items ints, kept at -1 between queries) maps item ->
// position in the query's target list, so cost is proportional to the
// contributions and the target list, never to n_items.

#include <algorithm>

#include "common.cuh"

namespace lk {

struct AccEnt {
    float w, v;
};

// heap order is reversed on weight (accum.rs:166-178): a <= b  <=>  b.w <= a.w
__device__ __forceinline__ bool ent_le(const AccEnt &a, const AccEnt &b) { return b.w <= a.w; }

__device__ void heap_sift_up(AccEnt *d, int start, int pos)
{
    AccEnt hole = d[pos];
    while (pos > start) {
        const int parent = (pos - 1) / 2;
        if (ent_le(hole, d[parent])) break;
        d[pos] = d[parent];
        pos = parent;
    }
    d[pos] = hole;
}

__device__ void heap_pop(AccEnt *d, int &len)
{
    AccEnt item = d[--len];
    if (len > 0) {
        AccEnt top = d[0];
        d[0] = item;
        item = top;
        // sift_down_to_bottom(0) then sift_up
        const int end = len;
        int pos = 0;
        AccEnt hole = d[0];
        int child = 1;
        while (end >= 2 && child <= end - 2) {
            if (ent_le(d[child], d[child + 1])) child += 1;
            d[pos] = d[child];
            pos = child;
            child = 2 * pos + 1;
        }
        if (child == end - 1) {
            d[pos] = d[child];
            pos = child;
        }
        d[pos] = hole;
        heap_sift_up(d, 0, pos);
    }
}

constexpr int SCORE_MAX_NBRS = 128;  // heap re-scoring keeps max_nbrs+1 entries in local memory

// One contribution into a ScoreAccumulator (accum.rs:86-117): vector until `limit` entries,
// then the Partial -> Full switch (pop from the back, push: accum.rs:73-82 — done in place by
// reversing the array and sifting the elements up one after the other, the same sequence of
// pushes), then Rust's BinaryHeap push / pop on the weight-reversed order.
__device__ void acc_push(AccEnt *d, int &len, int &is_heap, const AccEnt e, const int limit)
{
    if (!is_heap && len < limit) {
        d[len++] = e;
        return;
    }
    if (!is_heap) {
        const int n = len;
        for (int i = 0; i < n / 2; i++) {
            const AccEnt t = d[i];
            d[i] = d[n - 1 - i];
            d[n - 1 - i] = t;
        }
        for (int m = 1; m < n; m++) heap_sift_up(d, 0, m);
        is_heap = 1;
    }
    if (e.w > d[0].w) {  // accum.rs:107
        d[len++] = e;
        heap_sift_up(d, 0, len - 1);
        while (len > limit) heap_pop(d, len);
    }
}

// per-target heap state kept in the per-warp scratch of lk_knn_score_args::d_heap_scratch:
// [len, is_heap, (w, v) x (limit + 1)] as 32-bit words
__device__ __forceinline__ int heap_state_words(int limit) { return 2 + 2 * (limit + 1); }

// exact ScoreAccumulator replay for one (query, target) pair (fallback when the per-warp heap
// scratch is absent or full)
__device__ void rescore_exact(const lk_knn_score_args &a, int64_t r0, int64_t r1, int t, float *out_ws,
                              float *out_tw, int *out_len)
{
    AccEnt d[SCORE_MAX_NBRS + 1];
    int len = 0;
    int is_heap = 0;
    const int limit = a.max_nbrs;
    const int n_rows = a.user_mode ? a.n_matrix_rows : a.n_items;
    for (int64_t p = r0; p < r1; p++) {
        const int r = a.d_ref_items[p];
        if (r < 0 || r >= n_rows) continue;
        int64_t lo = a.d_sim_indptr[r], hi = a.d_sim_indptr[r + 1];
        const int64_t end = hi;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (a.d_sim_cols[mid] < t) lo = mid + 1; else hi = mid;
        }
        if (lo >= end || a.d_sim_cols[lo] != t) continue;
        const float mv = a.d_sim_vals ? a.d_sim_vals[lo] : 0.0f, hv = a.d_ref_vals ? a.d_ref_vals[p] : 0.0f;
        AccEnt e;
        e.w = a.user_mode ? hv : mv;
        e.v = a.user_mode ? mv : hv;
        acc_push(d, len, is_heap, e, limit);
    }
    float tw = 0.0f, ws = 0.0f;
    for (int i = 0; i < len; i++) tw = __fadd_rn(tw, d[i].w);
    for (int i = 0; i < len; i++) ws = __fadd_rn(ws, __fmul_rn(d[i].w, d[i].v));
    *out_ws = ws;
    *out_tw = tw;
    *out_len = len;
}

__global__ void __launch_bounds__(256) knn_score_kernel(lk_knn_score_args a)
{
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gwarp >= a.slotmap_warps) return;  // one slot-map row per working warp
    int32_t *slotmap = a.d_slotmap + (size_t)gwarp * a.n_items;
    // item mode: weight = similarity entry, value = the history entry's rating (item_score.rs:22-111);
    // user mode (user_score.rs:21-98): weight = the history entry's value (the neighbour's similarity),
    // value = the matrix entry (the neighbour's rating of the item)
    const bool user_mode = a.user_mode != 0;
    const int n_rows = user_mode ? a.n_matrix_rows : a.n_items;
    const bool explicit_fb = user_mode ? a.d_sim_vals != nullptr : a.d_ref_vals != nullptr;
    const float qnan = __int_as_float(0x7fc00000);
    const int hwords = heap_state_words(a.max_nbrs);
    uint32_t *heap_base = a.d_heap_scratch != nullptr
                              ? reinterpret_cast<uint32_t *>(a.d_heap_scratch) + (size_t)gwarp * a.heap_floats_per_warp
                              : nullptr;
    const int heap_cap = a.d_heap_scratch != nullptr ? (int)(a.heap_floats_per_warp / hwords) : 0;

    for (;;) {
        int q = 0;
        if (lane == 0) q = atomicAdd(a.d_work_counter, 1);
        q = __shfl_sync(FULL, q, 0);
        if (q >= a.n_queries) break;
        const int64_t t0 = a.d_tgt_indptr[q], t1 = a.d_tgt_indptr[q + 1];
        const int64_t r0 = a.d_ref_indptr[q], r1 = a.d_ref_indptr[q + 1];

        // 1. register the targets, zero their accumulator state
        for (int64_t x = t0 + lane; x < t1; x += 32) {
            const int t = a.d_tgt_items[x];
            a.d_acc_ws[x] = 0.0f;
            a.d_acc_tw[x] = 0.0f;
            a.d_acc_cnt[x] = 0;
            if (t >= 0 && t < a.n_items) slotmap[t] = (int32_t)(x - t0);
        }
        __syncwarp();

        // 2. contributions in history order; one similarity row's entries hit distinct targets
        for (int64_t p = r0; p < r1; p++) {
            const int r = a.d_ref_items[p];
            if (r < 0 || r >= n_rows) continue;  // null reference item (SURVEY.md App. A)
            const float hv = a.d_ref_vals ? a.d_ref_vals[p] : 0.0f;
            const int64_t s0 = a.d_sim_indptr[r], s1 = a.d_sim_indptr[r + 1];
            for (int64_t e = s0 + lane; e < s1; e += 32) {
                const int t = a.d_sim_cols[e];
                const int32_t slot = slotmap[t];
                if (slot >= 0) {
                    const float mv = a.d_sim_vals ? a.d_sim_vals[e] : 0.0f;
                    const float sim = user_mode ? hv : mv, rv = user_mode ? mv : hv;
                    if (sim != sim) atomicCAS(a.d_status, 0, 2);  // "similarity is null" (accum.rs:146-152)
                    const int64_t x = t0 + slot;
                    const int c = a.d_acc_cnt[x];
                    if (c < a.max_nbrs) {  // vector state: sums in push order
                        a.d_acc_tw[x] = __fadd_rn(a.d_acc_tw[x], sim);
                        if (explicit_fb) a.d_acc_ws[x] = __fadd_rn(a.d_acc_ws[x], __fmul_rn(sim, rv));
                    }
                    a.d_acc_cnt[x] = c + 1;
                }
            }
            __syncwarp();
        }

        // 2b. targets that received more than max_nbrs contributions have left the vector state:
        //     give each a heap in this warp's scratch (marker -(index+2) in its count) and run the
        //     history once more, every lane pushing its entry into its target's heap — the same
        //     element movement as the reference's accumulator, in the same order.  Targets that do
        //     not fit the scratch keep their count and are replayed one by one in step 3.
        if (heap_base != nullptr) {
            int n_tracked = 0;  // warp-uniform running count
            for (int64_t x0 = t0; x0 < t1; x0 += 32) {
                const int64_t x = x0 + lane;
                const bool over = x < t1 && a.d_acc_cnt[x] > a.max_nbrs;
                const unsigned m = __ballot_sync(FULL, over);
                if (m == 0u) continue;
                const int idx = n_tracked + __popc(m & ((1u << lane) - 1u));
                if (over && idx < heap_cap) {
                    a.d_acc_cnt[x] = -(idx + 2);
                    uint32_t *hs = heap_base + (size_t)idx * hwords;
                    hs[0] = 0u, hs[1] = 0u;
                }
                n_tracked += __popc(m);
            }
            __syncwarp();
            if (n_tracked > 0) {
                for (int64_t p = r0; p < r1; p++) {
                    const int r = a.d_ref_items[p];
                    if (r < 0 || r >= n_rows) continue;
                    const float hv = a.d_ref_vals ? a.d_ref_vals[p] : 0.0f;
                    const int64_t s0 = a.d_sim_indptr[r], s1 = a.d_sim_indptr[r + 1];
                    for (int64_t e = s0 + lane; e < s1; e += 32) {
                        const int32_t slot = slotmap[a.d_sim_cols[e]];
                        if (slot < 0) continue;
                        const int mk = a.d_acc_cnt[t0 + slot];
                        if (mk > -2) continue;
                        uint32_t *hs = heap_base + (size_t)(-mk - 2) * hwords;
                        int len = (int)hs[0], is_heap = (int)hs[1];
                        const float mv = a.d_sim_vals ? a.d_sim_vals[e] : 0.0f;
                        AccEnt ent;
                        ent.w = user_mode ? hv : mv;
                        ent.v = user_mode ? mv : hv;
                        acc_push(reinterpret_cast<AccEnt *>(hs + 2), len, is_heap, ent, a.max_nbrs);
                        hs[0] = (uint32_t)len, hs[1] = (uint32_t)is_heap;
                    }
                    __syncwarp();
                }
            }
        }

        // 3. finalise every target position (duplicate targets read the registered slot)
        for (int64_t x = t0 + lane; x < t1; x += 32) {
            const int t = a.d_tgt_items[x];
            float score = qnan;
            int count = -1;
            if (t >= 0 && t < a.n_items) {
                const int64_t xs = t0 + slotmap[t];
                int c = a.d_acc_cnt[xs];
                float ws = a.d_acc_ws[xs], tw = a.d_acc_tw[xs];
                if (c <= -2) {  // heap state built in step 2b: sums in heap-array order
                    const uint32_t *hs = heap_base + (size_t)(-c - 2) * hwords;
                    const AccEnt *d = reinterpret_cast<const AccEnt *>(hs + 2);
                    c = (int)hs[0];
                    tw = 0.0f, ws = 0.0f;
                    for (int i = 0; i < c; i++) tw = __fadd_rn(tw, d[i].w);
                    for (int i = 0; i < c; i++) ws = __fadd_rn(ws, __fmul_rn(d[i].w, d[i].v));
                } else if (c > a.max_nbrs) {
                    rescore_exact(a, r0, r1, t, &ws, &tw, &c);  // heap state, replayed from scratch
                }
                count = c;
                if (c >= a.min_nbrs) score = explicit_fb ? ws / tw : tw;
            }
            a.d_scores[x] = score;
            a.d_counts[x] = count;
        }
        __syncwarp();
        for (int64_t x = t0 + lane; x < t1; x += 32) {
            const int t = a.d_tgt_items[x];
            if (t >= 0 && t < a.n_items) slotmap[t] = -1;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// List-based variant (used when lk_knn_score_args::d_pool is given): no sequential walk over the
// history.  Contributions are counted per target with the 32 lanes working on 32 history entries at
// once, a prefix sum lays the targets' lists out in a pool, a second parallel pass fills the lists
// (chunks of 32 history entries are committed in order, so a list is sorted up to displacements
// inside one chunk), and every target then sorts its list by history position and replays it
// through the accumulator — vector sums in push order, BinaryHeap movement past max_nbrs — exactly
// as the sequential kernel does.  A query's cost no longer grows with the length of its history
// times a global-memory round trip.
// ---------------------------------------------------------------------------------------------
struct __align__(16) PoolEnt {
    int32_t pos;  // index of the reference item in the query's history
    float sim, rv;
    int32_t pad;
};

__global__ void __launch_bounds__(256) knn_score_lists_kernel(lk_knn_score_args a)
{
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gwarp >= a.slotmap_warps) return;  // one slot-map row per working warp
    int32_t *slotmap = a.d_slotmap + (size_t)gwarp * a.n_items;
    const bool user_mode = a.user_mode != 0;  // see knn_score_kernel
    const int n_rows = user_mode ? a.n_matrix_rows : a.n_items;
    const bool explicit_fb = user_mode ? a.d_sim_vals != nullptr : a.d_ref_vals != nullptr;
    const float qnan = __int_as_float(0x7fc00000);
    int32_t *acc_cnt = a.d_acc_cnt;
    int32_t *acc_off = reinterpret_cast<int32_t *>(a.d_acc_ws);  // list offset of a target (scratch reuse)
    int32_t *acc_cur = reinterpret_cast<int32_t *>(a.d_acc_tw);  // fill cursor of a target
    PoolEnt *pool = reinterpret_cast<PoolEnt *>(a.d_pool);
    const int limit = a.max_nbrs;

    for (;;) {
        int q = 0;
        if (lane == 0) q = atomicAdd(a.d_work_counter, 1);
        q = __shfl_sync(FULL, q, 0);
        if (q >= a.n_queries) break;
        const int64_t t0 = a.d_tgt_indptr[q], t1 = a.d_tgt_indptr[q + 1];
        const int64_t r0 = a.d_ref_indptr[q], r1 = a.d_ref_indptr[q + 1];

        // The passes over the target list (steps 1, 3, 5, 6) are latency-bound streams over per-query
        // arrays that live in DRAM: UB independent loads per lane are kept in flight.
        constexpr int UB = 8;

        // 1. register the targets
        for (int64_t xb = t0 + lane; xb < t1; xb += 32 * UB) {
            int tt[UB];
#pragma unroll
            for (int u = 0; u < UB; u++) tt[u] = xb + 32 * u < t1 ? __ldg(a.d_tgt_items + xb + 32 * u) : -1;
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = xb + 32 * u;
                if (x < t1) {
                    acc_cnt[x] = 0;
                    if (tt[u] >= 0 && tt[u] < a.n_items) slotmap[tt[u]] = (int32_t)(x - t0);
                }
            }
        }
        __syncwarp();

        // 2. count the contributions per target: one history entry per lane
        for (int64_t p0 = r0; p0 < r1; p0 += 32) {
            const int64_t p = p0 + lane;
            if (p < r1) {
                const int r = a.d_ref_items[p];
                if (r >= 0 && r < n_rows) {
                    const int64_t s1 = a.d_sim_indptr[r + 1];
                    for (int64_t e = a.d_sim_indptr[r]; e < s1; e += UB) {  // UB entries of the row in flight
                        int cc[UB], sl[UB];
                        float sv[UB];
                        const float hv = a.d_ref_vals ? a.d_ref_vals[p] : 0.0f;
#pragma unroll
                        for (int u = 0; u < UB; u++) {
                            cc[u] = e + u < s1 ? __ldg(a.d_sim_cols + e + u) : -1;
                            sv[u] = user_mode ? hv : ((e + u < s1 && a.d_sim_vals) ? __ldg(a.d_sim_vals + e + u) : 0.0f);
                        }
#pragma unroll
                        for (int u = 0; u < UB; u++) sl[u] = cc[u] >= 0 ? slotmap[cc[u]] : -1;
#pragma unroll
                        for (int u = 0; u < UB; u++) {
                            if (sl[u] >= 0) {
                                if (sv[u] != sv[u]) atomicCAS(a.d_status, 0, 2);  // "similarity is null"
                                atomicAdd(&acc_cnt[t0 + sl[u]], 1);
                            }
                        }
                    }
                }
            }
        }
        __syncwarp();

        // 3. lay the lists out: exclusive prefix sum of the counts, one pool segment per query
        int running = 0;
        for (int64_t x0 = t0; x0 < t1; x0 += 32 * UB) {
            int cc[UB];
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = x0 + 32 * u + lane;
                cc[u] = x < t1 ? __ldcg(&acc_cnt[x]) : 0;
            }
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = x0 + 32 * u + lane;
                const int incl = warp_incl_scan(cc[u], lane);
                if (x < t1) {
                    acc_off[x] = running + incl - cc[u];
                    acc_cur[x] = 0;
                }
                running += __shfl_sync(FULL, incl, 31);
            }
        }
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(a.d_pool_cursor, (unsigned long long)running);
        base = __shfl_sync(FULL, base, 0);
        const bool fits = base + (unsigned long long)running <= (unsigned long long)a.pool_entries;
        if (!fits && lane == 0) atomicCAS(a.d_status, 0, 3);  // pool too small (caller sizing error)
        __syncwarp();

        // 4. fill the lists; chunks of 32 history entries are committed in order
        if (fits) {
            for (int64_t p0 = r0; p0 < r1; p0 += 32) {
                const int64_t p = p0 + lane;
                if (p < r1) {
                    const int r = a.d_ref_items[p];
                    if (r >= 0 && r < n_rows) {
                        const float hv = a.d_ref_vals ? a.d_ref_vals[p] : 0.0f;
                        const int64_t s1 = a.d_sim_indptr[r + 1];
                        for (int64_t e = a.d_sim_indptr[r]; e < s1; e += UB) {
                            int cc[UB], sl[UB], of[UB], kp[UB];
                            float sv[UB];  // the matrix entry's value
#pragma unroll
                            for (int u = 0; u < UB; u++) {
                                cc[u] = e + u < s1 ? __ldg(a.d_sim_cols + e + u) : -1;
                                sv[u] = (e + u < s1 && a.d_sim_vals) ? __ldg(a.d_sim_vals + e + u) : 0.0f;
                            }
#pragma unroll
                            for (int u = 0; u < UB; u++) sl[u] = cc[u] >= 0 ? slotmap[cc[u]] : -1;
#pragma unroll
                            for (int u = 0; u < UB; u++) {
                                of[u] = sl[u] >= 0 ? acc_off[t0 + sl[u]] : 0;
                                kp[u] = sl[u] >= 0 ? atomicAdd(&acc_cur[t0 + sl[u]], 1) : 0;
                            }
#pragma unroll
                            for (int u = 0; u < UB; u++) {
                                if (sl[u] >= 0) {
                                    PoolEnt ent;
                                    ent.pos = (int32_t)(p - r0);
                                    ent.sim = user_mode ? hv : sv[u];
                                    ent.rv = user_mode ? sv[u] : hv;
                                    ent.pad = 0;
                                    pool[base + (unsigned long long)(of[u] + kp[u])] = ent;
                                }
                            }
                        }
                    }
                }
                __syncwarp();
            }
        }
        __threadfence_block();
        __syncwarp();

        // 5. every registered target sorts its list by history position and replays it; null targets
        //    are answered on the way, duplicates of a target are left for step 5b
        bool any_dup = false;
        for (int64_t xb = t0 + lane; xb < t1; xb += 32 * UB) {
            int tt[UB], sm[UB], nn[UB];
#pragma unroll
            for (int u = 0; u < UB; u++) tt[u] = xb + 32 * u < t1 ? __ldg(a.d_tgt_items + xb + 32 * u) : -1;
#pragma unroll
            for (int u = 0; u < UB; u++) sm[u] = (tt[u] >= 0 && tt[u] < a.n_items) ? slotmap[tt[u]] : -1;
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = xb + 32 * u;
                nn[u] = (fits && sm[u] >= 0 && t0 + sm[u] == x) ? __ldcg(&acc_cnt[x]) : 0;
            }
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = xb + 32 * u;
                if (x >= t1) continue;
                if (sm[u] < 0) {  // null (or out-of-range) target
                    a.d_scores[x] = qnan;
                    a.d_counts[x] = -1;
                    continue;
                }
                if (t0 + sm[u] != x) {
                    any_dup = true;
                    continue;
                }
                const int n = nn[u];
                float ws = 0.0f, tw = 0.0f;
                int c = n;
                if (n > 0) {
                    PoolEnt *L = pool + base + (unsigned long long)acc_off[x];
                    for (int i = 1; i < n; i++) {  // insertion sort: displacements stay inside a 32-entry chunk
                        const PoolEnt key = L[i];
                        int j = i - 1;
                        while (j >= 0 && L[j].pos > key.pos) {
                            L[j + 1] = L[j];
                            j--;
                        }
                        L[j + 1] = key;
                    }
                    if (n <= limit) {  // vector state: sums in push order (accum.rs:86-98, 196-231)
                        for (int i = 0; i < n; i++) tw = __fadd_rn(tw, L[i].sim);
                        if (explicit_fb)
                            for (int i = 0; i < n; i++) ws = __fadd_rn(ws, __fmul_rn(L[i].sim, L[i].rv));
                    } else {
                        AccEnt d[SCORE_MAX_NBRS + 1];
                        int len = 0, is_heap = 0;
                        for (int i = 0; i < n; i++) {
                            AccEnt ent;
                            ent.w = L[i].sim;
                            ent.v = L[i].rv;
                            acc_push(d, len, is_heap, ent, limit);
                        }
                        for (int i = 0; i < len; i++) tw = __fadd_rn(tw, d[i].w);
                        for (int i = 0; i < len; i++) ws = __fadd_rn(ws, __fmul_rn(d[i].w, d[i].v));
                        c = len;
                    }
                }
                a.d_counts[x] = c;
                a.d_scores[x] = (c >= a.min_nbrs) ? (explicit_fb ? ws / tw : tw) : qnan;
            }
        }
        __syncwarp();
        // 5b. duplicate targets copy the registered position's result (rare: skipped when there are none)
        if (__any_sync(FULL, any_dup)) {
            for (int64_t x = t0 + lane; x < t1; x += 32) {
                const int t = a.d_tgt_items[x];
                if (t >= 0 && t < a.n_items && t0 + slotmap[t] != x) {
                    a.d_scores[x] = a.d_scores[t0 + slotmap[t]];
                    a.d_counts[x] = a.d_counts[t0 + slotmap[t]];
                }
            }
            __syncwarp();
        }
        // 6. leave the slot map at -1
        for (int64_t xb = t0 + lane; xb < t1; xb += 32 * UB) {
            int tt[UB];
#pragma unroll
            for (int u = 0; u < UB; u++) tt[u] = xb + 32 * u < t1 ? __ldg(a.d_tgt_items + xb + 32 * u) : -1;
#pragma unroll
            for (int u = 0; u < UB; u++)
                if (tt[u] >= 0 && tt[u] < a.n_items) slotmap[tt[u]] = -1;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// Dense variant: every query is scored against ALL items (d_tgt_items == NULL; the batch runner's
// "score every candidate" case, the one the build+score metric is quoted on).  The list kernel above
// makes several passes over a query's whole target list — 59 k slots of which ~3 k ever receive a
// contribution — and needs a per-warp slot map; here the target of a contribution IS its output
// position.  A CTA per query; everything that is touched at random lives in a slot map of the CTA's own
// (one int per item, reused for every query the CTA handles, so it stays in L2) and in compact
// per-CTA arrays indexed by "touched target number"; the query's output rows are written exactly once:
//   1. count: the contributions of a chunk of the history are flattened over the 256 threads (row extents
//      in shared memory, block scan, one binary search per contribution) and counted with atomics on the
//      slot map; a target touched for the first time joins the list of touched targets (shared memory,
//      spilling into the query's own — still unwritten — count row);
//   2. layout: block scan over the touched targets' counts gives every list its offset in the contribution
//      pool; the slot map entry becomes the touched-target number;
//   3. fill: the same flattened walk appends (history position, weight, value) to the lists;
//   4. replay: one thread per touched target sorts its list by history position and runs it through the
//      accumulator (vector sums in push order / BinaryHeap movement past max_nbrs) — the same bits as the
//      sequential walk;
//   5. one coalesced pass writes the score and count rows — the result where the slot map has an entry,
//      NaN / 0 elsewhere — and clears the slot map for the next query.
// (Round-2 v2 counted on the output row itself and kept [n_queries x n_items] offset / cursor rows: 2.1 MB
// of DRAM traffic per ML-25M-shaped query, twice its output, L2 hit rate 28 %.)
// ---------------------------------------------------------------------------------------------
constexpr int DENSE_THREADS = 256;
constexpr int DENSE_ACTIVE_CAP = 8192;  // touched targets kept in shared memory (the rest: the query's count row)
constexpr int DENSE_HIST_CHUNK = 2048;  // history entries flattened at a time

struct DenseSmem {
    int32_t active[DENSE_ACTIVE_CAP];
    long long row0[DENSE_HIST_CHUNK];  // first matrix entry of the history entry's row
    int32_t pre[DENSE_HIST_CHUNK + 1];  // exclusive prefix of the row lengths
    float hv[DENSE_HIST_CHUNK];         // the history entry's value
};

__device__ __forceinline__ int block_excl_scan(int v, int *s_scan, int *s_carry, int tid, int lane, int warp)
{
    // exclusive scan of v over the block, continuing from *s_carry; returns this thread's offset and advances the carry
    const int incl = warp_incl_scan(v, lane);
    if (lane == 31) s_scan[warp] = incl;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < warp; w++) woff += s_scan[w];
    const int carry = *s_carry;
    __syncthreads();
    if (tid == DENSE_THREADS - 1) *s_carry = carry + woff + incl;
    __syncthreads();
    return carry + woff + incl - v;
}

__global__ void __launch_bounds__(DENSE_THREADS) knn_score_dense_kernel(lk_knn_score_args a)
{
    extern __shared__ __align__(16) unsigned char dense_raw[];
    DenseSmem &sm = *reinterpret_cast<DenseSmem *>(dense_raw);
    __shared__ int s_scan[DENSE_THREADS / 32];
    __shared__ int s_q, s_nactive, s_carry;
    __shared__ unsigned long long s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool user_mode = a.user_mode != 0;
    const int n_rows = user_mode ? a.n_matrix_rows : a.n_items;
    const bool explicit_fb = user_mode ? a.d_sim_vals != nullptr : a.d_ref_vals != nullptr;
    const float qnan = __int_as_float(0x7fc00000);
    const int limit = a.max_nbrs;
    const int64_t NI = a.n_items;
    PoolEnt *pool = reinterpret_cast<PoolEnt *>(a.d_pool);
    // per-CTA state, reused by every query this CTA handles
    int32_t *slot = a.d_slotmap + (size_t)blockIdx.x * NI;  // all zero between queries
    int32_t *offs = reinterpret_cast<int32_t *>(a.d_acc_ws) + (size_t)blockIdx.x * NI;  // [touched target] list offset, later score bits
    int32_t *curs = reinterpret_cast<int32_t *>(a.d_acc_tw) + (size_t)blockIdx.x * NI;  // [touched target] list cursor, later count
    constexpr int CU = 4;  // contributions per thread and step of the flattened walk

    for (;;) {
        if (tid == 0) {
            s_q = atomicAdd(a.d_work_counter, 1);
            s_nactive = 0;
        }
        __syncthreads();
        if (s_q >= a.n_queries) break;
        const int q = a.d_deferred ? a.d_deferred[s_q] : s_q;  // optional hand-out order (heaviest queries first)
        const int64_t r0 = a.d_ref_indptr[q], r1 = a.d_ref_indptr[q + 1];
        float *scores = a.d_scores + (int64_t)q * NI;
        int32_t *counts = a.d_counts + (int64_t)q * NI;
        // the query's count row is not written before step 5: until then it holds the tail of the touched list
        auto active_at = [&](int i) { return i < DENSE_ACTIVE_CAP ? sm.active[i] : __ldcg(&counts[i - DENSE_ACTIVE_CAP]); };

        // walk over the contributions of the query, flattened over the block:
        // fn(lo, tcol, mval, pos0) gets four contributions per thread and step — lo[u] = history entry inside
        // the chunk (-1: none), its matrix column and value, pos0 = history position of the chunk — with the
        // matrix entries already loaded; the callers stage their own atomics the same way (all issued before
        // any result is used): the walk is bound by memory latency, not by bandwidth
        auto for_each_contribution = [&](auto fn) {
            for (int64_t h0 = r0; h0 < r1; h0 += DENSE_HIST_CHUNK) {
                const int nh = (int)min((int64_t)DENSE_HIST_CHUNK, r1 - h0);
                if (tid == 0) s_carry = 0;
                __syncthreads();
                for (int i0 = 0; i0 < nh; i0 += DENSE_THREADS) {
                    const int i = i0 + tid;
                    int len = 0;
                    if (i < nh) {
                        const int r = a.d_ref_items[h0 + i];
                        long long e0 = 0;
                        if (r >= 0 && r < n_rows) {  // null / unknown reference items contribute nothing
                            e0 = a.d_sim_indptr[r];
                            len = (int)(a.d_sim_indptr[r + 1] - e0);
                        }
                        sm.row0[i] = e0;
                        sm.hv[i] = a.d_ref_vals ? a.d_ref_vals[h0 + i] : 0.0f;
                    }
                    const int off = block_excl_scan(len, s_scan, &s_carry, tid, lane, warp);
                    if (i < nh) sm.pre[i] = off;
                }
                if (tid == 0) sm.pre[nh] = s_carry;
                __syncthreads();
                const int total = sm.pre[nh];
                for (int c0 = tid; c0 < total; c0 += DENSE_THREADS * CU) {
                    int lo[CU], tcol[CU];
                    float mval[CU];
#pragma unroll
                    for (int u = 0; u < CU; u++) {
                        const int c = c0 + u * DENSE_THREADS;
                        lo[u] = -1;
                        tcol[u] = 0;
                        mval[u] = 0.0f;
                        if (c < total) {
                            int l = 0, hi = nh;  // last i with pre[i] <= c
                            while (hi - l > 1) {
                                const int mid = (l + hi) >> 1;
                                if (sm.pre[mid] <= c) l = mid; else hi = mid;
                            }
                            lo[u] = l;
                            const long long e = sm.row0[l] + (c - sm.pre[l]);
                            tcol[u] = __ldg(a.d_sim_cols + e);
                            if (a.d_sim_vals) mval[u] = __ldg(a.d_sim_vals + e);
                        }
                    }
                    fn(lo, tcol, mval, (int)(h0 - r0));
                }
                __syncthreads();
            }
        };

        // 1. count
        for_each_contribution([&](const int (&lo)[CU], const int (&tcol)[CU], const float (&mval)[CU], int) {
            int old[CU];
            bool null_w = false;
#pragma unroll
            for (int u = 0; u < CU; u++) {
                old[u] = 1;
                if (lo[u] >= 0) {
                    const float w = user_mode ? sm.hv[lo[u]] : mval[u];
                    null_w |= w != w;
                    old[u] = atomicAdd(&slot[tcol[u]], 1);
                }
            }
            if (null_w) atomicCAS(a.d_status, 0, 2);  // "similarity is null" (accum.rs:146-152)
#pragma unroll
            for (int u = 0; u < CU; u++) {
                if (old[u] == 0) {  // first touch of this target
                    const int idx = atomicAdd(&s_nactive, 1);
                    if (idx < DENSE_ACTIVE_CAP) sm.active[idx] = tcol[u]; else __stcg(&counts[idx - DENSE_ACTIVE_CAP], tcol[u]);
                }
            }
        });
        __threadfence_block();
        __syncthreads();
        const int n_active = s_nactive;

        // 2. lay out the lists: block-wide exclusive scan of the touched targets' counts; slot -> touched-target number
        if (tid == 0) s_carry = 0;
        __syncthreads();
        for (int i0 = 0; i0 < n_active; i0 += DENSE_THREADS) {
            const int i = i0 + tid;
            const int t = i < n_active ? active_at(i) : 0;
            const int c = i < n_active ? __ldcg(&slot[t]) : 0;
            const int off = block_excl_scan(c, s_scan, &s_carry, tid, lane, warp);
            if (i < n_active) {
                __stcg(&offs[i], off);
                __stcg(&curs[i], 0);
                __stcg(&slot[t], i + 1);
            }
        }
        const int total = s_carry;
        if (tid == 0) s_base = atomicAdd(a.d_pool_cursor, (unsigned long long)total);
        __threadfence_block();
        __syncthreads();
        const unsigned long long base = s_base;
        if (base + (unsigned long long)total > (unsigned long long)a.pool_entries) {
            if (tid == 0) atomicCAS(a.d_status, 0, 3);  // pool too small (caller sizing error)
            for (int i = tid; i < n_active; i += DENSE_THREADS) __stcg(&slot[active_at(i)], 0);  // leave the map clean
            __syncthreads();
            continue;
        }

        // 3. fill the lists (arrival order; sorted per target below)
        for_each_contribution([&](const int (&lo)[CU], const int (&tcol)[CU], const float (&mval)[CU], int pos0) {
            int ti[CU], kpos[CU], off[CU];
#pragma unroll
            for (int u = 0; u < CU; u++) ti[u] = lo[u] >= 0 ? __ldcg(&slot[tcol[u]]) - 1 : -1;
#pragma unroll
            for (int u = 0; u < CU; u++) {
                kpos[u] = 0, off[u] = 0;
                if (ti[u] >= 0) {
                    kpos[u] = atomicAdd(&curs[ti[u]], 1);
                    off[u] = __ldcg(&offs[ti[u]]);
                }
            }
#pragma unroll
            for (int u = 0; u < CU; u++) {
                if (ti[u] >= 0) {
                    const float hv = sm.hv[lo[u]];
                    PoolEnt ent;
                    ent.pos = pos0 + lo[u];
                    ent.sim = user_mode ? hv : mval[u];
                    ent.rv = user_mode ? mval[u] : hv;
                    ent.pad = 0;
                    pool[base + (unsigned long long)(off[u] + kpos[u])] = ent;
                }
            }
        });
        __threadfence_block();
        __syncthreads();

        // 4. one thread per touched target: history order, then the accumulator
        constexpr int RU = 4;
        for (int i0 = tid; i0 < n_active; i0 += DENSE_THREADS * RU) {
          int nn[RU], oo[RU];
#pragma unroll
          for (int v = 0; v < RU; v++) {
              const int i = i0 + v * DENSE_THREADS;
              nn[v] = i < n_active ? __ldcg(&curs[i]) : 0;
              oo[v] = i < n_active ? __ldcg(&offs[i]) : 0;
          }
#pragma unroll 1
          for (int v = 0; v < RU; v++) {
            const int i = i0 + v * DENSE_THREADS;
            if (i >= n_active) break;
            const int n = nn[v];
            PoolEnt *L = pool + base + (unsigned long long)oo[v];
            for (int u = 1; u < n; u++) {  // insertion sort by history position
                const PoolEnt key = L[u];
                int j = u - 1;
                while (j >= 0 && L[j].pos > key.pos) {
                    L[j + 1] = L[j];
                    j--;
                }
                L[j + 1] = key;
            }
            float ws = 0.0f, tw = 0.0f;
            int c = n;
            if (n <= limit) {  // vector state: sums in push order (accum.rs:86-98, 196-231)
                for (int u = 0; u < n; u++) tw = __fadd_rn(tw, L[u].sim);
                if (explicit_fb)
                    for (int u = 0; u < n; u++) ws = __fadd_rn(ws, __fmul_rn(L[u].sim, L[u].rv));
            } else {
                AccEnt d[SCORE_MAX_NBRS + 1];
                int len = 0, is_heap = 0;
                for (int u = 0; u < n; u++) {
                    AccEnt ent;
                    ent.w = L[u].sim;
                    ent.v = L[u].rv;
                    acc_push(d, len, is_heap, ent, limit);
                }
                for (int u = 0; u < len; u++) tw = __fadd_rn(tw, d[u].w);
                for (int u = 0; u < len; u++) ws = __fadd_rn(ws, __fmul_rn(d[u].w, d[u].v));
                c = len;
            }
            __stcg(&curs[i], c);
            __stcg(&offs[i], __float_as_int(c >= a.min_nbrs ? (explicit_fb ? ws / tw : tw) : qnan));
          }
        }
        __threadfence_block();
        __syncthreads();

        // 5. the output rows, once, coalesced; the slot map goes back to zero
        constexpr int FU = 8;
        for (int64_t x0 = tid; x0 < NI; x0 += DENSE_THREADS * FU) {
            int sl[FU];
#pragma unroll
            for (int u = 0; u < FU; u++) {
                const int64_t x = x0 + u * DENSE_THREADS;
                sl[u] = x < NI ? __ldcg(&slot[x]) : 0;
            }
#pragma unroll
            for (int u = 0; u < FU; u++) {
                const int64_t x = x0 + u * DENSE_THREADS;
                if (x >= NI) break;
                float sc = qnan;
                int ct = 0;
                if (sl[u] != 0) {
                    sc = __int_as_float(__ldcg(&offs[sl[u] - 1]));
                    ct = __ldcg(&curs[sl[u] - 1]);
                    __stcg(&slot[x], 0);
                }
                __stcs(&scores[x], sc);
                __stcs(&counts[x], ct);
            }
        }
        __syncthreads();
    }
}

constexpr int SCORE_WARPS_PER_SM = 16;

}  // namespace lk

using namespace lk;

extern "C" {

int64_t lk_knn_score_warps(void) { return (int64_t)sm_count() * SCORE_WARPS_PER_SM; }

int64_t lk_knn_score_dense_ctas(void) { return (int64_t)sm_count() * 3; }

int lk_knn_score_batch(const lk_knn_score_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_knn_score_batch: null args");
    const lk_knn_score_args &a = *args;
    LK_REQUIRE(a.n_items >= 1 && a.n_queries >= 0, LK_ERR_INVALID, "bad shape");
    LK_REQUIRE(a.max_nbrs >= 1 && a.max_nbrs <= SCORE_MAX_NBRS, LK_ERR_UNSUPPORTED,
               "max_nbrs must be in 1..%d", SCORE_MAX_NBRS);
    const bool dense = a.d_tgt_items == nullptr && a.d_tgt_indptr == nullptr;  // every query against all items
    LK_REQUIRE(a.d_sim_indptr && a.d_sim_cols && a.d_ref_indptr && a.d_ref_items && a.d_acc_ws && a.d_acc_tw &&
                   a.d_scores && a.d_counts && a.d_work_counter && a.d_status,
               LK_ERR_INVALID, "lk_knn_score_batch: null pointer");
    LK_REQUIRE(dense || (a.d_tgt_indptr && a.d_tgt_items && a.d_slotmap && a.d_acc_cnt), LK_ERR_INVALID,
               "lk_knn_score_batch: null pointer (target lists)");
    LK_REQUIRE(!dense || (a.d_pool && a.d_pool_cursor && a.d_slotmap && a.slotmap_warps >= lk_knn_score_dense_ctas()),
               LK_ERR_INVALID,
               "lk_knn_score_batch: the dense (all-items) mode needs the contribution pool and one n_items row of "
               "d_slotmap per CTA (lk_knn_score_dense_ctas)");
    LK_REQUIRE(a.user_mode ? a.d_ref_vals != nullptr : a.d_sim_vals != nullptr, LK_ERR_INVALID,
               "lk_knn_score_batch: the weights (similarities) are missing");
    LK_REQUIRE(dense || a.slotmap_warps >= 1, LK_ERR_INVALID, "slotmap too small");
    if (a.n_queries == 0) return LK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    if (dense) {
        LK_REQUIRE(reinterpret_cast<uintptr_t>(a.d_pool) % 16 == 0 && a.pool_entries >= 0, LK_ERR_INVALID,
                   "lk_knn_score_batch: bad contribution pool");
        LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
        // the per-CTA slot maps (n_items ints each) should stay in L2 next to the similarity matrix: two CTAs
        // per SM instead of three when three rows per SM would take more than half of it
        const Options &opt = options();
        int per_sm = ((int64_t)sm_count() * 3 * a.n_items * 4 > (int64_t)(64 << 20)) ? 2 : 3;
        if (opt.knn_score_ctas > 0) per_sm = std::min(3, opt.knn_score_ctas);
        const int grid = (int)std::min<int64_t>(a.n_queries, (int64_t)sm_count() * per_sm);
        const int smem = (int)sizeof(DenseSmem);
        LK_CUDA_TRY(cudaFuncSetAttribute(knn_score_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        knn_score_dense_kernel<<<grid, DENSE_THREADS, smem, st>>>(a);
        LK_CUDA_TRY(cudaGetLastError());
        return LK_OK;
    }
    // as many warps as there are slot-map rows (the caller sizes them to the batch), at most the full grid
    const int64_t warps = std::min<int64_t>(a.slotmap_warps, lk_knn_score_warps());
    const int blocks = (int)((warps + 7) / 8);
    // with a contribution pool the list-based kernel runs (LK_KNN_SCORE_SEQ=1 forces the sequential one)
    if (a.d_pool != nullptr && a.d_pool_cursor != nullptr && options().knn_score_seq != 1) {
        LK_REQUIRE(reinterpret_cast<uintptr_t>(a.d_pool) % 16 == 0 && a.pool_entries >= 0, LK_ERR_INVALID,
                   "lk_knn_score_batch: bad contribution pool");
        LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
        knn_score_lists_kernel<<<blocks, 256, 0, st>>>(a);
    } else {
        knn_score_kernel<<<blocks, 256, 0, st>>>(a);
    }
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
