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
//     order;
//   * a target that receives more than `max_nbrs` contributions switches to a
//     min-heap (accum.rs:73-82,100-117), emulated with the Rust std BinaryHeap
//     element movement so that the survivor set under ties and the summation
//     order match;
//   * null (negative) reference items are skipped, null targets give NaN / -1.
//
// Neither kernel walks the history one entry after the other.  The contributions
// of a query are counted and scattered in parallel into one list per target in a
// contribution pool; each list is then sorted by history position and replayed
// through the accumulator by one thread (replay_list), which restores the order
// the reference sees.
//   * knn_score_lists_kernel (explicit target lists): one warp owns one query.  A
//     per-warp `slotmap` (n_items ints, kept at -1 between queries) maps item ->
//     position in the query's target list, so cost is proportional to the
//     contributions and the target list, never to n_items.
//   * knn_score_dense_kernel (every query against all items): one CTA per query.  Its ranking mode
//     (lk_knn_recommend_batch) replaces the full output rows by each query's top n, selected in the kernel.

#include <algorithm>

#include "common.cuh"
#include "topn_heap.cuh"

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

// ---------------------------------------------------------------------------------------------
// Target-list kernel: the contributions are counted per target with the 32 lanes working on 32 history
// entries at once, a prefix sum lays the targets' lists out in the pool, a second parallel pass fills the
// lists (chunks of 32 history entries are committed in order, so a list is sorted up to displacements
// inside one chunk), and every target then replays its list (replay_list).  A query's cost does not grow
// with the length of its history times a global-memory round trip.
// ---------------------------------------------------------------------------------------------
struct __align__(16) PoolEnt {
    int32_t pos;  // index of the reference item in the query's history
    float sim, rv;
    int32_t pad;
};

// One target's contribution list [n entries] through a ScoreAccumulator: sorted by history position in
// place (insertion sort: the lists arrive nearly sorted), then summed in push order while it fits the vector
// state (accum.rs:86-98, 196-231), or replayed through the BinaryHeap movement past `limit` and summed in
// heap-array order.  Returns the accumulator's length; ws is only summed with explicit feedback.
__device__ __forceinline__ int replay_list(PoolEnt *L, const int n, const int limit, const bool explicit_fb,
                                           float &ws, float &tw)
{
    for (int i = 1; i < n; i++) {
        const PoolEnt key = L[i];
        int j = i - 1;
        while (j >= 0 && L[j].pos > key.pos) {
            L[j + 1] = L[j];
            j--;
        }
        L[j + 1] = key;
    }
    ws = 0.0f, tw = 0.0f;
    if (n <= limit) {
        for (int i = 0; i < n; i++) tw = __fadd_rn(tw, L[i].sim);
        if (explicit_fb)
            for (int i = 0; i < n; i++) ws = __fadd_rn(ws, __fmul_rn(L[i].sim, L[i].rv));
        return n;
    }
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
    return len;
}

__global__ void __launch_bounds__(256) knn_score_lists_kernel(lk_knn_score_args a)
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
    int32_t *list_cnt = a.d_list_cnt, *list_off = a.d_list_off, *list_cur = a.d_list_cur;
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
                    list_cnt[x] = 0;
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
                                atomicAdd(&list_cnt[t0 + sl[u]], 1);
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
                cc[u] = x < t1 ? __ldcg(&list_cnt[x]) : 0;
            }
#pragma unroll
            for (int u = 0; u < UB; u++) {
                const int64_t x = x0 + 32 * u + lane;
                const int incl = warp_incl_scan(cc[u], lane);
                if (x < t1) {
                    list_off[x] = running + incl - cc[u];
                    list_cur[x] = 0;
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
                                of[u] = sl[u] >= 0 ? list_off[t0 + sl[u]] : 0;
                                kp[u] = sl[u] >= 0 ? atomicAdd(&list_cur[t0 + sl[u]], 1) : 0;
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
                nn[u] = (fits && sm[u] >= 0 && t0 + sm[u] == x) ? __ldcg(&list_cnt[x]) : 0;
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
                float ws = 0.0f, tw = 0.0f;
                int c = 0;
                if (nn[u] > 0)
                    c = replay_list(pool + base + (unsigned long long)list_off[x], nn[u], limit, explicit_fb, ws, tw);
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
//      accumulator (replay_list, as in the list kernel);
//   5. one coalesced pass writes the score and count rows — the result where the slot map has an entry,
//      NaN / 0 elsewhere — and clears the slot map for the next query.
// Ranking mode (RANK, lk_knn_recommend_batch) keeps steps 1-4 and replaces step 5 by rank_query below: the
// query's top n of its final scores, written as n entries instead of two n_items rows.
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

// ---------------------------------------------------------------------------------------------
// Ranking mode.  For every query the result must be the reference's per-query composition
//     cands = all items ascending, minus the excluded ones;  il = scorer(query, cands);  il[argtopn(il.scores, n)]
// argtopn (sorting.rs:131-170, topn.cu) offers the candidates in index order to an indirect min-heap and returns
// on a NaN offer before it touches the heap.  So offering EVERY item in ascending item order, with the excluded
// and the untouched items as NaN, replays the reference's heap move for move; its keys are item numbers.
//   * the offer order is the item order of the slot-map walk, never the touched list (atomic arrival order);
//   * the only pre-filter is the heap root once the heap is full: the root never decreases after that and a full
//     heap rejects s <= root.  A filter against a guessed n-th score would change which equal scores survive;
//   * the offsets are added in f32 before ranking, as the components add them to the scores on the host.
// The CTA walks the slot-map row in chunks of RANK_CHUNK items (coalesced, clearing the map as step 5 does),
// compacts the candidates that pass the filter in item order (ballots and a 64-entry scan) and one thread offers
// them to the heap of topn_heap.cuh.  The heap and the candidate buffer live in DenseSmem, which steps 1-3 no
// longer need at that point, so the ranking mode costs no shared memory of its own.
// ---------------------------------------------------------------------------------------------
constexpr int RANK_UNITS = 8;    // items per thread and chunk
constexpr int RANK_CHUNK = DENSE_THREADS * RANK_UNITS;
constexpr int RANK_WARPS = DENSE_THREADS / 32;

struct RankSmem {
    float hv[TOPN_MAX];  // heap: score, item number, accumulator length
    int32_t hk[TOPN_MAX];
    int32_t hc[TOPN_MAX];
    float cv[RANK_CHUNK];  // the chunk's candidates, in item order
    int32_t ck[RANK_CHUNK];
    int32_t cc[RANK_CHUNK];
    int32_t wcnt[RANK_UNITS * RANK_WARPS];  // candidates per (unit, warp); then their exclusive offsets
    int32_t wofs[RANK_UNITS * RANK_WARPS];
    int32_t n_cand, count;
    float root;
};
static_assert(sizeof(RankSmem) <= sizeof(DenseSmem), "the ranking state must fit in the dense kernel's shared memory");

// the ranking heap in RankSmem; its entries carry the accumulator length beside the item number
struct RankHeap {
    struct Ent {
        float v;
        int32_t k, c;
    };
    RankSmem &r;
    __device__ __forceinline__ float val(const int p) const { return r.hv[p]; }
    __device__ __forceinline__ Ent get(const int p) const { return {r.hv[p], r.hk[p], r.hc[p]}; }
    __device__ __forceinline__ void put(const int p, const Ent e) { r.hv[p] = e.v, r.hk[p] = e.k, r.hc[p] = e.c; }
};

// Ranking mode's step 5 for query q (the whole CTA; steps 1-4 done, DenseSmem free): exclusion, the ranking walk,
// the heap sort and the n output entries.  Leaves the slot map at zero.
__device__ void rank_query(RankSmem &r, const lk_knn_rank_args &rk, const int q, int32_t *slot, int32_t *offs,
                           const int32_t *curs, const int64_t NI, const int n_active, const int tid, const int lane,
                           const int warp)
{
    const float qnan = __int_as_float(0x7fc00000);
    const int n = rk.n;
    // items never recommended to the query: their touched target's score becomes NaN
    if (rk.d_excl_indptr != nullptr) {
        const int64_t e1 = rk.d_excl_indptr[q + 1];
        for (int64_t p = rk.d_excl_indptr[q] + tid; p < e1; p += DENSE_THREADS) {
            const int e = rk.d_excl_items[p];
            if (e >= 0 && e < NI) {
                const int sl = __ldcg(&slot[e]);
                if (sl != 0) __stcg(&offs[sl - 1], __float_as_int(qnan));
            }
        }
    }
    if (tid == 0) r.count = 0;
    __threadfence_block();
    __syncthreads();
    const float qoff = rk.d_query_offset != nullptr ? rk.d_query_offset[q] : 0.0f;
    const unsigned lanes_below = (1u << lane) - 1u;
    // no touched target: every score is NaN and the slot map is already clean
    for (int64_t x0 = 0; n_active > 0 && x0 < NI; x0 += RANK_CHUNK) {
        const int count0 = r.count;  // the heap as the previous chunk left it
        const float root0 = r.root;
        int sl[RANK_UNITS];
#pragma unroll
        for (int u = 0; u < RANK_UNITS; u++) {
            const int64_t x = x0 + u * DENSE_THREADS + tid;
            sl[u] = x < NI ? __ldcg(&slot[x]) : 0;
        }
        float sv[RANK_UNITS];
        int32_t sc[RANK_UNITS];
        unsigned pass[RANK_UNITS];
#pragma unroll
        for (int u = 0; u < RANK_UNITS; u++) {
            const int64_t x = x0 + u * DENSE_THREADS + tid;
            float s = qnan;
            sc[u] = 0;
            if (sl[u] != 0) {
                s = __int_as_float(__ldcg(&offs[sl[u] - 1]));
                sc[u] = __ldcg(&curs[sl[u] - 1]);
                __stcg(&slot[x], 0);
                if (rk.d_item_offset != nullptr) s = __fadd_rn(s, rk.d_item_offset[x]);
                if (rk.d_query_offset != nullptr) s = __fadd_rn(s, qoff);
            }
            sv[u] = s;
            pass[u] = __ballot_sync(FULL, s == s && (count0 < n || s > root0));
        }
        if (lane == 0)
#pragma unroll
            for (int u = 0; u < RANK_UNITS; u++) r.wcnt[u * RANK_WARPS + warp] = __popc(pass[u]);
        __syncthreads();
        static_assert(RANK_UNITS * RANK_WARPS == 64, "one warp scans the (unit, warp) counts two per lane");
        if (warp == 0) {
            const int c0 = r.wcnt[2 * lane], c1 = r.wcnt[2 * lane + 1];
            const int incl = warp_incl_scan(c0 + c1, lane);
            r.wofs[2 * lane] = incl - c0 - c1;
            r.wofs[2 * lane + 1] = incl - c1;
            if (lane == 31) r.n_cand = incl;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < RANK_UNITS; u++) {
            if (pass[u] >> lane & 1u) {
                const int p = r.wofs[u * RANK_WARPS + warp] + __popc(pass[u] & lanes_below);
                r.cv[p] = sv[u];
                r.ck[p] = (int32_t)(x0 + u * DENSE_THREADS + tid);
                r.cc[p] = sc[u];
            }
        }
        __syncthreads();
        if (tid == 0 && r.n_cand > 0) {
            int count = count0;
            float root = root0;
            const int nc = r.n_cand;
            RankHeap h{r};
            for (int i = 0; i < nc; i++) topn_heap_offer(h, count, root, n, RankHeap::Ent{r.cv[i], r.ck[i], r.cc[i]});
            r.count = count;
            r.root = root;
        }
        __syncthreads();
    }
    // heap.rs:56-65 topn_vec: heap sort into descending score order
    const int count = r.count;
    if (tid == 0) {
        RankHeap h{r};
        topn_heap_sort(h, count);
    }
    __syncthreads();
    const int64_t o = (int64_t)q * n;
    for (int t = tid; t < n; t += DENSE_THREADS) {
        const bool in = t < count;
        rk.d_out_idx[o + t] = in ? r.hk[t] : -1;
        rk.d_out_val[o + t] = in ? r.hv[t] : qnan;
        rk.d_out_nbrs[o + t] = in ? r.hc[t] : 0;
    }
    if (tid == 0) rk.d_out_cnt[q] = count;
}

template <bool RANK>
__global__ void __launch_bounds__(DENSE_THREADS) knn_score_dense_kernel(lk_knn_score_args a, lk_knn_rank_args rk)
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
    int32_t *offs = a.d_list_off + (size_t)blockIdx.x * NI;  // [touched target] list offset, later score bits
    int32_t *curs = a.d_list_cur + (size_t)blockIdx.x * NI;  // [touched target] list cursor, later count
    constexpr int CU = 4;  // contributions per thread and step of the flattened walk

    for (;;) {
        if (tid == 0) {
            s_q = atomicAdd(a.d_work_counter, 1);
            s_nactive = 0;
        }
        __syncthreads();
        if (s_q >= a.n_queries) break;
        const int q = s_q;
        const int64_t r0 = a.d_ref_indptr[q], r1 = a.d_ref_indptr[q + 1];
        float *scores = RANK ? nullptr : a.d_scores + (int64_t)q * NI;
        int32_t *counts = RANK ? nullptr : a.d_counts + (int64_t)q * NI;
        // the tail of the touched list: the query's count row, not written before step 5; in ranking mode, which
        // has no such row, the CTA's own spill row
        int32_t *spill = RANK ? rk.d_spill + (size_t)blockIdx.x * NI : counts;
        auto active_at = [&](int i) { return i < DENSE_ACTIVE_CAP ? sm.active[i] : __ldcg(&spill[i - DENSE_ACTIVE_CAP]); };

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
                    if (idx < DENSE_ACTIVE_CAP) sm.active[idx] = tcol[u]; else __stcg(&spill[idx - DENSE_ACTIVE_CAP], tcol[u]);
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
            float ws, tw;
            const int c = replay_list(pool + base + (unsigned long long)oo[v], nn[v], limit, explicit_fb, ws, tw);
            __stcg(&curs[i], c);
            __stcg(&offs[i], __float_as_int(c >= a.min_nbrs ? (explicit_fb ? ws / tw : tw) : qnan));
          }
        }
        __threadfence_block();
        __syncthreads();

        if constexpr (RANK) {
            // q and n_active re-read from shared memory: kept in registers across step 4 they cost a spill
            rank_query(*reinterpret_cast<RankSmem *>(dense_raw), rk, s_q, slot, offs, curs, NI, s_nactive, tid, lane,
                       warp);
            __syncthreads();
            continue;
        }
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

}  // extern "C"

// The checks lk_knn_score_batch and lk_knn_recommend_batch share.  `outputs`: d_scores / d_counts are required.
static int check_score_args(const lk_knn_score_args &a, const char *who, const bool outputs)
{
    LK_REQUIRE(a.n_items >= 1 && a.n_queries >= 0, LK_ERR_INVALID, "bad shape");
    LK_REQUIRE(a.max_nbrs >= 1 && a.max_nbrs <= SCORE_MAX_NBRS, LK_ERR_UNSUPPORTED,
               "max_nbrs must be in 1..%d", SCORE_MAX_NBRS);
    const bool dense = a.d_tgt_items == nullptr && a.d_tgt_indptr == nullptr;  // every query against all items
    LK_REQUIRE(a.d_sim_indptr && a.d_sim_cols && a.d_ref_indptr && a.d_ref_items && a.d_list_off && a.d_list_cur &&
                   (!outputs || (a.d_scores && a.d_counts)) && a.d_work_counter && a.d_status,
               LK_ERR_INVALID, "%s: null pointer", who);
    LK_REQUIRE(a.d_pool && a.d_pool_cursor, LK_ERR_INVALID,
               "%s: the contribution pool (d_pool, d_pool_cursor) is required", who);
    LK_REQUIRE(reinterpret_cast<uintptr_t>(a.d_pool) % 16 == 0 && a.pool_entries >= 0, LK_ERR_INVALID,
               "%s: bad contribution pool", who);
    LK_REQUIRE(dense || (a.d_tgt_indptr && a.d_tgt_items && a.d_slotmap && a.d_list_cnt), LK_ERR_INVALID,
               "%s: null pointer (target lists)", who);
    LK_REQUIRE(!dense || (a.d_slotmap && a.slotmap_warps >= lk_knn_score_dense_ctas()), LK_ERR_INVALID,
               "%s: the dense (all-items) mode needs one n_items row of d_slotmap per CTA "
               "(lk_knn_score_dense_ctas)", who);
    LK_REQUIRE(a.user_mode ? a.d_ref_vals != nullptr : a.d_sim_vals != nullptr, LK_ERR_INVALID,
               "%s: the weights (similarities) are missing", who);
    LK_REQUIRE(dense || a.slotmap_warps >= 1, LK_ERR_INVALID, "slotmap too small");
    return LK_OK;
}

template <bool RANK>
static int launch_dense(const lk_knn_score_args &a, const lk_knn_rank_args &rk, cudaStream_t st)
{
    // the per-CTA slot maps (n_items ints each) should stay in L2 next to the similarity matrix: two CTAs
    // per SM instead of three when three rows per SM would take more than half of it
    const Options &opt = options();
    int per_sm = ((int64_t)sm_count() * 3 * a.n_items * 4 > (int64_t)(64 << 20)) ? 2 : 3;
    if (opt.knn_score_ctas > 0) per_sm = std::min(3, opt.knn_score_ctas);
    const int grid = (int)std::min<int64_t>(a.n_queries, (int64_t)sm_count() * per_sm);
    const int smem = (int)sizeof(DenseSmem);
    LK_CUDA_TRY(
        cudaFuncSetAttribute(knn_score_dense_kernel<RANK>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    knn_score_dense_kernel<RANK><<<grid, DENSE_THREADS, smem, st>>>(a, rk);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

extern "C" {

int lk_knn_score_batch(const lk_knn_score_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_knn_score_batch: null args");
    const lk_knn_score_args &a = *args;
    const int rc = check_score_args(a, "lk_knn_score_batch", true);
    if (rc != LK_OK) return rc;
    const bool dense = a.d_tgt_items == nullptr && a.d_tgt_indptr == nullptr;
    if (a.n_queries == 0) return LK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
    if (dense) return launch_dense<false>(a, lk_knn_rank_args{}, st);
    // as many warps as there are slot-map rows (the caller sizes them to the batch), at most the full grid
    const int64_t warps = std::min<int64_t>(a.slotmap_warps, lk_knn_score_warps());
    const int blocks = (int)((warps + 7) / 8);
    knn_score_lists_kernel<<<blocks, 256, 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_knn_recommend_batch(const lk_knn_score_args *score, const lk_knn_rank_args *rank, void *stream)
{
    LK_REQUIRE(score != nullptr && rank != nullptr, LK_ERR_INVALID, "lk_knn_recommend_batch: null args");
    const lk_knn_score_args &a = *score;
    const lk_knn_rank_args &rk = *rank;
    const int rc = check_score_args(a, "lk_knn_recommend_batch", false);
    if (rc != LK_OK) return rc;
    LK_REQUIRE(a.d_tgt_items == nullptr && a.d_tgt_indptr == nullptr, LK_ERR_INVALID,
               "lk_knn_recommend_batch: ranks all items (dense mode: d_tgt_indptr and d_tgt_items must be NULL)");
    LK_REQUIRE(rk.n >= 1 && rk.n <= TOPN_MAX, LK_ERR_UNSUPPORTED, "lk_knn_recommend_batch: n must be in 1..%d",
               TOPN_MAX);
    LK_REQUIRE(rk.d_spill && rk.d_out_idx && rk.d_out_val && rk.d_out_nbrs && rk.d_out_cnt, LK_ERR_INVALID,
               "lk_knn_recommend_batch: null pointer (spill rows or outputs)");
    LK_REQUIRE(rk.d_excl_indptr == nullptr || rk.d_excl_items != nullptr, LK_ERR_INVALID,
               "lk_knn_recommend_batch: d_excl_items is required with d_excl_indptr");
    if (a.n_queries == 0) return LK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
    return launch_dense<true>(a, rk, st);
}

}  // extern "C"
