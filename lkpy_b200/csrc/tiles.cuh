// tiles.cuh — the tiled sparse-accumulation core of the item-kNN build (knn_build.cu), the user-kNN search
// (knn_user.cu), the co-occurrence count and association scoring (cooc.cu).
//
// Each of them builds output rows as sums of sparse rows: a CTA of W warps owns one column tile of the output row
// in shared memory, warp w the sub-tile [w * TW, (w + 1) * TW) of it, and tile pointers give the segment of every
// input row that falls into a sub-tile.  A warp walks the input rows 32 at a time, flattening their segments over
// the lanes for the loads (warp_walk_segments), and applies the entries one input row per round
// (warp_apply_in_owner_order), so every accumulator receives its additions from one warp, in input-row order.
// Survivors of a unit go to one bump-allocated pool segment (cta_emit_pool_segment), and pool_to_csr_kernel
// gathers the segments into a row-sorted CSR.
#pragma once

#include "common.cuh"

namespace lk {

// The CTA's next work index from `counter` (INT_MAX once the optional cancel flag is raised).  `slot` is shared
// memory; all threads of the CTA must call.
__device__ __forceinline__ int cta_next_work(int32_t *counter, const int32_t *cancel, int *slot)
{
    if (threadIdx.x == 0) *slot = fetch_work(counter, cancel);
    __syncthreads();
    const int wi = *slot;
    __syncthreads();
    return wi;
}

// The entries of the sub-tile segments of up to 32 input rows, lane r holding row r's segment (source index
// `base`, `len` entries, 0 for a lane past the last row), flattened over the lanes 32 at a time.  Every round
// calls body(e_valid, owner, src): this lane's entry, if e_valid, is at source index `src` and belongs to the
// row of lane `owner` (the caller shuffles its per-row payload from there).  Idx is the type of the source
// index.  Returns whether the rows had any entry.  All lanes of the warp must call.
template <typename Idx, typename Body>
__device__ __forceinline__ bool warp_walk_segments(Idx base, int len, int lane, Body body)
{
    const int incl = warp_incl_scan(len, lane);
    const int total = __shfl_sync(FULL, incl, 31);
    const Idx adj = base - (incl - len);  // source index = adj[owner] + e
    for (int e0 = 0; e0 < total; e0 += 32) {
        const int e = e0 + lane;
        int own = 0;  // owner: smallest lane with incl > e
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const int t = __shfl_sync(FULL, incl, own + step - 1);
            if (t <= e) own += step;
        }
        own = min(own, 31);
        body(e < total, own, __shfl_sync(FULL, adj, own) + e);
    }
    return total > 0;
}

// fn() on every valid lane, one owner per round in ascending lane order: the lanes of one owner (input row) touch
// distinct columns, so each accumulator gets its additions in input-row order.
// (Grouping lanes by column instead — __match_any_sync, or one ballot per column bit — was measured slower on
// ML-25M-shaped data: a popular column is present in most users' segments, so the rounds per batch stay near the
// number of users.)
template <typename Fn>
__device__ __forceinline__ void warp_apply_in_owner_order(bool valid, int owner, Fn fn)
{
    unsigned pend = __ballot_sync(FULL, valid);
    while (pend) {
        const int leader_owner = __shfl_sync(FULL, owner, __ffs(pend) - 1);  // every lane shuffles
        const bool mine = valid && owner == leader_owner;
        if (mine) fn();
        __syncwarp();
        pend &= ~__ballot_sync(FULL, mine);
    }
}

// One pool segment for work unit `unit`: every warp counts the accumulators v of its sub-tile `my` (columns col0 +
// [0, TW)) with keep(v, col), 32 at a time (ballot + popcount keep column order); the CTA bump-allocates the
// segment from *cursor, or raises *status to 1 and writes nothing when the pool of `capacity` entries is full; the
// warps write (col, bits(v, col)) in column order and reset their accumulators to `reset`.  wcnt: W ints of
// shared memory.  All threads of the CTA must call.
template <int W, typename T, typename Keep, typename Bits>
__device__ __forceinline__ void cta_emit_pool_segment(T *my, int TW, int col0, int64_t unit, Keep keep, Bits bits,
                                                      T reset, int *wcnt, unsigned long long *cursor,
                                                      int64_t capacity, int32_t *status, int64_t *pool_off,
                                                      int32_t *part_cnt, int32_t *pool_cols, uint32_t *pool_vals)
{
    __shared__ unsigned long long s_off;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int cnt = 0;
    for (int c0 = 0; c0 < TW; c0 += 32) cnt += __popc(__ballot_sync(FULL, keep(my[c0 + lane], col0 + c0 + lane)));
    if (lane == 0) wcnt[warp] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        for (int w = 0; w < W; w++) n += wcnt[w];
        unsigned long long off = atomicAdd(cursor, (unsigned long long)n);
        if (off + (unsigned long long)n > (unsigned long long)capacity) {
            atomicCAS(status, 0, 1);
            off = ~0ull;
        }
        s_off = off;
        pool_off[unit] = (int64_t)off;
        part_cnt[unit] = n;
    }
    __syncthreads();
    const unsigned long long off = s_off;
    int pos = 0;
    for (int w = 0; w < warp; w++) pos += wcnt[w];
    for (int c0 = 0; c0 < TW; c0 += 32) {
        const int c = col0 + c0 + lane;
        const T v = my[c0 + lane];
        const bool k = keep(v, c);
        const unsigned b = __ballot_sync(FULL, k);
        if (k && off != ~0ull) {
            const unsigned long long at = off + pos + __popc(b & ((1u << lane) - 1u));
            pool_cols[at] = c;
            pool_vals[at] = bits(v, c);
        }
        pos += __popc(b);
        my[c0 + lane] = reset;
    }
    __syncthreads();  // wcnt and s_off are rewritten by the next unit
}

// One warp per output row: copies the pool segments of the row's units [row * units_per_row, (row + 1) *
// units_per_row), in that order, to the row of the CSR.  V is the 32-bit value type of the pool.
template <typename V>
__global__ void pool_to_csr_kernel(int n_rows, int units_per_row, const int64_t *__restrict__ pool_off,
                                   const int32_t *__restrict__ part_cnt, const int32_t *__restrict__ pool_cols,
                                   const V *__restrict__ pool_vals, const int64_t *__restrict__ out_indptr,
                                   int32_t *__restrict__ out_cols, V *__restrict__ out_vals)
{
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n_rows; row += warps) {
        int64_t dst = out_indptr[row];
        for (int64_t u = (int64_t)row * units_per_row; u < (int64_t)(row + 1) * units_per_row; u++) {
            const int64_t src = pool_off[u];
            const int c = part_cnt[u];
            for (int t = lane; t < c; t += 32) {
                out_cols[dst + t] = pool_cols[src + t];
                out_vals[dst + t] = pool_vals[src + t];
            }
            dst += c;
        }
    }
}

template <typename V>
int launch_pool_to_csr(int n_rows, int units_per_row, const int64_t *pool_off, const int32_t *part_cnt,
                       const int32_t *pool_cols, const V *pool_vals, const int64_t *out_indptr, int32_t *out_cols,
                       V *out_vals, void *stream)
{
    pool_to_csr_kernel<V><<<sm_count() * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        n_rows, units_per_row, pool_off, part_cnt, pool_cols, pool_vals, out_indptr, out_cols, out_vals);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

// Column tiling of an n_cols-wide accumulator row for `warps` sub-tiles per CTA and `ctas` CTAs per SM: the
// fewest column tiles ("halves") of warps * tile_cols columns, tile_cols a multiple of 32, whose acc_bytes-wide
// accumulators fit the shared memory of a CTA (227 KB usable per SM, 1 KB reserved per CTA) next to its
// fixed_bytes and `reserve` bytes of headroom.  n_cols >= 1.
inline void tile_geometry(int32_t n_rows, int32_t n_cols, int warps, int ctas, int acc_bytes, int fixed_bytes,
                          int reserve, lk_knn_geom *geom)
{
    const int max_cols = ((227 * 1024) / ctas - 1024 - fixed_bytes - reserve) / acc_bytes;
    const int64_t halves = ((int64_t)n_cols + max_cols - 1) / max_cols;
    const int cw = (int)((n_cols + halves - 1) / halves);
    int tw = (cw + warps - 1) / warps;
    tw = (tw + 31) & ~31;
    while ((int64_t)tw * warps > max_cols && tw > 32) tw -= 32;
    geom->n_users = n_rows;
    geom->n_items = n_cols;
    geom->warps = warps;
    geom->tile_cols = tw;
    geom->n_halves = (int)(((int64_t)n_cols + tw * warps - 1) / (tw * warps));
    geom->n_subtiles = geom->n_halves * warps;
    geom->smem_bytes = warps * tw * acc_bytes + fixed_bytes;
    geom->ctas_per_sm = ctas;
}

}  // namespace lk
