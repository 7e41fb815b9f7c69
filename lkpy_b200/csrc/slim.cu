// slim.cu — SLIM / fsSLIM training for sm_90a: one elastic-net weight column per target item by coordinate
// descent, bit for bit what train_slim computes (src/accel/slim/mod.rs:57-93, compute_column and below).
//
// A persistent grid hands out target columns, most expensive first, to single warps.  Each warp owns a slice of a
// global-memory workspace, kept zero between columns: resid [n_users] f32, W [n_items] f32 (the reference's
// dense weights vector), pc [n_items] int32 (path counts), and two int32 [n_items] item lists (the active set and
// the radix sort's second buffer).  Per column:
//   * active set: the target's users' UI rows are walked 32 entries at a time in stored order (the tile core's
//     warp_walk_segments).  Lanes holding the same item find each other with __match_any_sync; the lowest adds
//     the group's size to pc and, when pc was 0, the item is a first encounter, appended in lane order (ballot +
//     prefix popcount), i.e. in first-encounter order.
//   * fsSLIM (max_nbrs < |active|): a stable LSD radix sort of the active list on the 64-bit ordered bits of the
//     f64 key -(pc)/(sqrt(|U_i|) sqrt(|U_j|)), recomputed from pc and the IU offsets in every pass, then
//     truncation — exactly the reference's stable sort_by_key + resize.
//   * coordinate descent: every lane forms t = resid[u] + w for its user independently (one rounding each), the 32
//     values go through shared memory and every lane adds them in user order onto upd (the strictly sequential f32
//     chain of the reference; invalid lanes contribute -0.0, which adds nothing).  The soft threshold and the
//     resid -= diff stores follow; diff == +0 leaves every residual unchanged and skips the stores.
//   * output: the W entries >= 1e-12 are counted over the visited coordinates, one pool segment is bump-allocated,
//     and W is swept in ascending item order with ballots to write (j, W[j]); a full pool raises the status word
//     and writes nothing.  Then every touched workspace entry is reset to zero.
// lk_slim_pool_to_csr gathers the segments with the shared pool_to_csr_kernel.
#include "tiles.cuh"

namespace lk {

constexpr int SL_WARPS = 8;
constexpr int SL_NT = SL_WARPS * 32;
constexpr int SL_CTAS = 4;  // resident CTAs per SM (<= 64 registers)
constexpr float SL_EPSILON = 1.0e-12f;
constexpr float SL_TOLERANCE = 1e-3f;

__host__ __device__ inline int64_t sl_align(int64_t b) { return (b + 255) & ~int64_t(255); }

__host__ __device__ inline int64_t sl_warp_bytes(int32_t n_users, int32_t n_items)
{
    return sl_align((int64_t)n_users * 4) + 4 * sl_align((int64_t)n_items * 4);
}

static inline int64_t sl_ctas(int64_t n_work)
{
    const int64_t want = (n_work + SL_WARPS - 1) / SL_WARPS;
    const int64_t most = (int64_t)sm_count() * SL_CTAS;
    return want < most ? want : most;
}

// the f64 fsSLIM key of mod.rs:250-254 as order-preserving bits: ascending bits = ascending keys
__device__ __forceinline__ uint64_t sl_key_bits(int pc, int nj, double i_norm)
{
    const double key = __ddiv_rn(-(double)pc, __dmul_rn(i_norm, __dsqrt_rn((double)nj)));
    const uint64_t b = (uint64_t)__double_as_longlong(key);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__global__ void __launch_bounds__(SL_NT, SL_CTAS) slim_train_kernel(const lk_slim_args a)
{
    __shared__ __align__(16) float s_t[SL_WARPS][32];
    __shared__ int s_hist[SL_WARPS][256];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    float *t_s = s_t[wib];
    int *hist = s_hist[wib];

    const int64_t gw = (int64_t)blockIdx.x * SL_WARPS + wib;
    unsigned char *ws = static_cast<unsigned char *>(a.d_workspace) + gw * sl_warp_bytes(a.n_users, a.n_items);
    float *resid = reinterpret_cast<float *>(ws);
    float *W = reinterpret_cast<float *>(ws + sl_align((int64_t)a.n_users * 4));
    const int64_t ib = sl_align((int64_t)a.n_items * 4);
    int32_t *pc = reinterpret_cast<int32_t *>(reinterpret_cast<unsigned char *>(W) + ib);
    int32_t *active = reinterpret_cast<int32_t *>(reinterpret_cast<unsigned char *>(pc) + ib);
    int32_t *spare = reinterpret_cast<int32_t *>(reinterpret_cast<unsigned char *>(active) + ib);

    const int32_t *ui_ptr = a.d_ui_indptr, *ui_cols = a.d_ui_cols, *iu_ptr = a.d_iu_indptr, *iu_cols = a.d_iu_cols;

    for (;;) {
        int wi = 0;
        if (lane == 0) wi = fetch_work(a.d_work_counter, a.d_cancel);
        wi = __shfl_sync(FULL, wi, 0);
        if (wi >= a.n_work) break;
        const int item = a.d_sched[wi];
        const int i0 = iu_ptr[item], ni = iu_ptr[item + 1] - i0;

        // residuals and the active set in first-encounter order (mod.rs:216-232)
        int n_act = 0;
        for (int t0 = 0; t0 < ni; t0 += 32) {
            int base = 0, len = 0;
            if (t0 + lane < ni) {
                const int u = __ldg(iu_cols + i0 + t0 + lane);
                resid[u] = 1.0f;
                base = __ldg(ui_ptr + u);
                len = __ldg(ui_ptr + u + 1) - base;
            }
            warp_walk_segments(base, len, lane, [&](bool valid, int, int src) {
                const int j = valid ? __ldg(ui_cols + src) : -1;
                const bool cand = valid && j != item;
                const unsigned peers = __match_any_sync(FULL, cand ? j : -1 - lane);
                const bool leader = cand && (peers & lt) == 0;
                int old = 1;
                if (leader) {
                    old = pc[j];
                    pc[j] = old + __popc(peers);
                }
                const unsigned first = __ballot_sync(FULL, old == 0);
                if (old == 0) active[n_act + __popc(first & lt)] = j;
                n_act += __popc(first);
                __syncwarp();
            });
        }

        // fsSLIM: stable sort by the cosine key, keep the first k (mod.rs:234-256)
        const int32_t *order = active;
        int n_cd = n_act;
        if (a.max_nbrs >= 0 && a.max_nbrs < n_act) {
            const double i_norm = __dsqrt_rn((double)ni);
            int32_t *src = active, *dst = spare;
            auto digit = [&](int j, int shift) {
                const int nj = __ldg(iu_ptr + j + 1) - __ldg(iu_ptr + j);
                return (int)((sl_key_bits(pc[j], nj, i_norm) >> shift) & 255u);
            };
            for (int shift = 0; shift < 64; shift += 8) {
                __syncwarp();
                for (int b = lane; b < 256; b += 32) hist[b] = 0;
                __syncwarp();
                for (int p = lane; p < n_act; p += 32) atomicAdd(&hist[digit(src[p], shift)], 1);
                __syncwarp();
                int v[8], s = 0;
                bool all_one = false;
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    v[q] = hist[lane * 8 + q];
                    all_one |= v[q] == n_act;
                    s += v[q];
                }
                if (__any_sync(FULL, all_one)) continue;  // one digit for every key: the pass moves nothing
                int run = warp_incl_scan(s, lane) - s;
                __syncwarp();
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    hist[lane * 8 + q] = run;
                    run += v[q];
                }
                __syncwarp();
                for (int p0 = 0; p0 < n_act; p0 += 32) {
                    const int p = p0 + lane;
                    const bool valid = p < n_act;
                    int j = 0, d = 256 + lane;
                    if (valid) {
                        j = src[p];
                        d = digit(j, shift);
                    }
                    const unsigned peers = __match_any_sync(FULL, d);
                    const int rank = __popc(peers & lt);
                    const int at = valid ? hist[d] : 0;
                    __syncwarp();
                    if (valid) {
                        dst[at + rank] = j;
                        if (rank == 0) hist[d] = at + __popc(peers);
                    }
                    __syncwarp();
                }
                int32_t *t = src;
                src = dst;
                dst = t;
            }
            __syncwarp();
            order = src;
            n_cd = a.max_nbrs;
        }

        // coordinate descent (mod.rs:259-320)
        for (int it = 0; it < a.max_iters; it++) {
            float dmax = 0.0f;
            for (int c = 0; c < n_cd; c++) {
                const int j = order[c];
                const int p0 = __ldg(iu_ptr + j), nj = __ldg(iu_ptr + j + 1) - p0;
                const float w = W[j];
                float upd = 0.0f;
                for (int t0 = 0; t0 < nj; t0 += 32) {
                    float t = -0.0f;
                    if (t0 + lane < nj) t = __fadd_rn(resid[__ldg(iu_cols + p0 + t0 + lane)], w);
                    t_s[lane] = t;
                    __syncwarp();
                    const float4 *t4 = reinterpret_cast<const float4 *>(t_s);
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        const float4 x = t4[q];
                        upd = __fadd_rn(upd, x.x);
                        upd = __fadd_rn(upd, x.y);
                        upd = __fadd_rn(upd, x.z);
                        upd = __fadd_rn(upd, x.w);
                    }
                    __syncwarp();
                }
                float nw = 0.0f;
                if (upd >= a.l1_reg) nw = __fdiv_rn(__fsub_rn(upd, a.l1_reg), __fadd_rn(__int2float_rn(nj), a.l2_reg));
                const float diff = __fsub_rn(nw, w);
                __syncwarp();  // every lane has read W[j]
                if (lane == 0) W[j] = nw;
                if (diff != 0.0f) {
                    for (int t = lane; t < nj; t += 32) {
                        const int u = __ldg(iu_cols + p0 + t);
                        resid[u] = __fsub_rn(resid[u], diff);
                    }
                }
                __syncwarp();
                const float ad = fabsf(diff);
                if (ad > dmax) dmax = ad;
            }
            if (dmax <= SL_TOLERANCE) break;
        }

        // output: every W[j] >= 1e-12 in ascending j (mod.rs:168-178)
        int cnt = 0;
        for (int c0 = 0; c0 < n_cd; c0 += 32) {
            const bool keep = c0 + lane < n_cd && W[order[c0 + lane]] >= SL_EPSILON;
            cnt += __popc(__ballot_sync(FULL, keep));
        }
        unsigned long long off = 0;
        if (lane == 0) {
            off = atomicAdd(a.d_pool_cursor, (unsigned long long)cnt);
            if (off + (unsigned long long)cnt > (unsigned long long)a.pool_capacity) {
                atomicCAS(a.d_status, 0, 1);
                off = ~0ull;
            }
            a.d_pool_off[item] = (int64_t)off;
            a.d_part_cnt[item] = cnt;
        }
        off = __shfl_sync(FULL, off, 0);
        if (off != ~0ull) {
            int pos = 0;
            for (int j0 = 0; pos < cnt; j0 += 32) {
                const int j = j0 + lane;
                const float v = j < a.n_items ? W[j] : 0.0f;
                const bool keep = v >= SL_EPSILON;
                const unsigned b = __ballot_sync(FULL, keep);
                if (keep) {
                    const unsigned long long at = off + pos + __popc(b & lt);
                    a.d_pool_cols[at] = j;
                    a.d_pool_vals[at] = v;
                }
                pos += __popc(b);
            }
        }
        __syncwarp();

        // reset the touched workspace: W and the residuals of the visited coordinates, the target's residuals,
        // the path counts of the whole active set
        for (int c0 = 0; c0 < n_cd; c0 += 32) {
            int base = 0, len = 0;
            if (c0 + lane < n_cd) {
                const int j = order[c0 + lane];
                W[j] = 0.0f;
                base = __ldg(iu_ptr + j);
                len = __ldg(iu_ptr + j + 1) - base;
            }
            warp_walk_segments(base, len, lane, [&](bool valid, int, int src) {
                if (valid) resid[__ldg(iu_cols + src)] = 0.0f;
            });
        }
        for (int t = lane; t < ni; t += 32) resid[__ldg(iu_cols + i0 + t)] = 0.0f;
        for (int p = lane; p < n_act; p += 32) pc[order[p]] = 0;
        __syncwarp();
    }
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_slim_workspace_bytes(int32_t n_users, int32_t n_items, int64_t n_work, int64_t *bytes)
{
    LK_REQUIRE(n_users >= 0 && n_items >= 1 && n_work >= 0 && bytes != nullptr, LK_ERR_INVALID,
               "lk_slim_workspace_bytes: bad arguments");
    *bytes = sl_ctas(n_work) * SL_WARPS * sl_warp_bytes(n_users, n_items);
    return LK_OK;
}

static int slim_check(const lk_slim_args *args, const char *who)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "%s: null args", who);
    const lk_slim_args &a = *args;
    LK_REQUIRE(a.n_users >= 0 && a.n_items >= 1, LK_ERR_INVALID, "%s: bad shape", who);
    LK_REQUIRE(a.d_pool_off && a.d_part_cnt, LK_ERR_INVALID, "%s: null pool offsets", who);
    return LK_OK;
}

int lk_slim_train(const lk_slim_args *args, void *stream)
{
    if (int rc = slim_check(args, "lk_slim_train")) return rc;
    const lk_slim_args &a = *args;
    LK_REQUIRE(a.d_ui_indptr && a.d_ui_cols && a.d_iu_indptr && a.d_iu_cols, LK_ERR_INVALID,
               "lk_slim_train: null matrix");
    LK_REQUIRE(a.max_iters >= 0 && a.max_nbrs >= -1, LK_ERR_INVALID, "lk_slim_train: bad max_iters / max_nbrs");
    LK_REQUIRE(a.d_work_counter && a.d_status && a.d_pool_cursor, LK_ERR_INVALID, "lk_slim_train: null counter");
    LK_REQUIRE(a.n_work >= 0 && a.n_work <= a.n_items, LK_ERR_INVALID, "lk_slim_train: n_work must be <= n_items");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_status, 0, sizeof(int32_t), st));
    LK_CUDA_TRY(cudaMemsetAsync(a.d_pool_cursor, 0, sizeof(unsigned long long), st));
    if (a.n_work == 0) return LK_OK;
    LK_REQUIRE(a.d_sched && a.d_workspace && a.d_pool_cols && a.d_pool_vals, LK_ERR_INVALID,
               "lk_slim_train: null pointer");
    const int64_t ctas = sl_ctas(a.n_work);
    LK_REQUIRE(a.workspace_bytes >= ctas * SL_WARPS * sl_warp_bytes(a.n_users, a.n_items), LK_ERR_INVALID,
               "lk_slim_train: workspace smaller than lk_slim_workspace_bytes");
    slim_train_kernel<<<(unsigned)ctas, SL_NT, 0, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_slim_pool_to_csr(const lk_slim_args *args, const int64_t *d_out_indptr, int32_t *d_out_cols, float *d_out_vals,
                        void *stream)
{
    if (int rc = slim_check(args, "lk_slim_pool_to_csr")) return rc;
    LK_REQUIRE(d_out_indptr && d_out_cols && d_out_vals, LK_ERR_INVALID, "lk_slim_pool_to_csr: null output");
    const lk_slim_args &a = *args;
    return launch_pool_to_csr(a.n_items, 1, a.d_pool_off, a.d_part_cnt, a.d_pool_cols,
                              reinterpret_cast<const uint32_t *>(a.d_pool_vals), d_out_indptr, d_out_cols,
                              reinterpret_cast<uint32_t *>(d_out_vals), stream);
}

}  // extern "C"
