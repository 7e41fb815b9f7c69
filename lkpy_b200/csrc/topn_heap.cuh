// topn_heap.cuh — the one device copy of argtopn's indirect min-heap (src/accel/indirect/heap.rs,
// src/accel/data/sorting.rs:131-170) and of its output contract, shared by every batched top-n kernel: topn.cu,
// the ranking mode of knn_score.cu, als_recommend.cu, cooc.cu, ease.cu, basic.cu and stochastic.cu (f64 keys).
//
// The contract: candidates are offered in ascending item order, an excluded item counts as a NaN offer (never
// accepted), and each query's row of n is written in descending score order, padded with -1 items and NaN scores,
// beside its count.
//
// The heap is reached through a storage policy H so that each kernel keeps its own layout (per-thread local
// arrays, shared memory, a strided workspace) and its own payload:
//     typename H::Ent         the entry: a score `v` (float, or double for stochastic.cu's f64 keys) and whatever
//                             rides along with it
//     V     H::val(int pos)   the score at pos, of the type of `v`
//     Ent   H::get(int pos)   the entry at pos
//     void  H::put(int pos, Ent e)
// Both sifts move a hole instead of swapping, which leaves exactly the arrangement the reference's swaps leave.
#pragma once

namespace lk {

constexpr int TOPN_MAX = 1024;  // the largest n of every top-n entry point: lk_topn_max()

// (score, item) entries, entry p at hv[p * STRIDE] and hk[p * STRIDE] (STRIDE > 1 interleaves several heaps)
template <int STRIDE>
struct PairHeap {
    struct Ent {
        float v;
        int32_t k;
    };
    float *hv;
    int32_t *hk;
    __device__ __forceinline__ float val(const int p) const { return hv[p * STRIDE]; }
    __device__ __forceinline__ Ent get(const int p) const { return {hv[p * STRIDE], hk[p * STRIDE]}; }
    __device__ __forceinline__ void put(const int p, const Ent e) { hv[p * STRIDE] = e.v, hk[p * STRIDE] = e.k; }
};

// heap.rs:67-89 downheap: the smaller child, the left one on a tie, while strictly smaller than the moving entry
template <class H>
__device__ __forceinline__ void topn_heap_down(H &h, int pos, const int lim)
{
    const typename H::Ent e = h.get(pos);
    for (;;) {
        int mn = pos;
        auto mv = e.v;
        const int left = 2 * pos + 1, right = 2 * pos + 2;
        if (left < lim) {
            const auto lv = h.val(left);
            if (lv < mv) {
                mn = left;
                mv = lv;
            }
        }
        if (right < lim && h.val(right) < mv) mn = right;
        if (mn == pos) break;
        h.put(pos, h.get(mn));
        pos = mn;
    }
    h.put(pos, e);
}

// argtopn's offer of a non-NaN entry (the caller drops NaN, sorting.rs:142): heap.rs:41-45 push + upheap while
// the heap has room, else heap.rs:46-52 replace the root if strictly greater and downheap.  `root` mirrors the
// root's score once the heap holds an entry; V is the score type.
template <class H, typename V>
__device__ __forceinline__ void topn_heap_offer(H &h, int &count, V &root, const int n,
                                                const typename H::Ent e)
{
    if (count < n) {
        int pos = count++;
        while (pos > 0) {
            const int parent = (pos - 1) / 2;
            if (!(h.val(parent) > e.v)) break;
            h.put(pos, h.get(parent));
            pos = parent;
        }
        h.put(pos, e);
        root = h.val(0);
    } else if (e.v > root) {
        h.put(0, e);
        topn_heap_down(h, 0, n);
        root = h.val(0);
    }
}

// heap.rs:56-65 topn_vec: heap sort; positions 0..count-1 end up in descending score order
template <class H>
__device__ __forceinline__ void topn_heap_sort(H &h, const int count)
{
    for (int m = count - 1; m > 0; m--) {
        const typename H::Ent t = h.get(0);
        h.put(0, h.get(m));
        h.put(m, t);
        topn_heap_down(h, 0, m);
    }
}

// whether item is among the query's ascending exclusions ex[ec .. ee), advancing the cursor ec past smaller items;
// items are asked in ascending order, and an excluded item is argtopn's NaN offer
__device__ __forceinline__ bool topn_excluded(const int32_t *ex, int64_t &ec, const int64_t ee, const int item)
{
    while (ec < ee && ex[ec] < item) ec++;
    return ec < ee && ex[ec] == item;
}

}  // namespace lk
