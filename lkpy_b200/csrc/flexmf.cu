// flexmf.cu — gradient-trained matrix factorisation: FlexMFImplicitScorer (logistic and pairwise/BPR loss over sampled
// negatives) and FlexMFExplicitScorer (squared error on centred ratings, no negatives): the negative sampler and one
// minibatch step (forward, loss, per-row gradient sums, Adam update).
//
// A step is four launches on the caller's stream:
//   flexmf_forward_kernel   one warp per sample: the scores of the positive and the n negatives (n = 0 for MSE), dL/ds
//                           of each (coef [B][1+n]) and the sample's share of the loss;
//   flexmf_loss_kernel      one block adds the B shares in a fixed order (f64) into d_loss[0];
//   flexmf_grad_kernel      one warp per unit.  The occurrences of a row in the batch are sorted by position and cut
//                           into units of at most 64, so that a row that fills half the batch is spread over the
//                           grid; a unit adds its occurrences in order into partials[unit] from the tables as they
//                           were BEFORE this step (nothing has been updated yet);
//   flexmf_update_kernel    one thread per (row, 4 columns): adds the row's unit partials in unit order and applies
//                           AdamW to every row (dense) or SparseAdam to the rows of the batch, in place.
// The gradient and the update are separate launches because a user row's gradient reads the item rows of the same
// batch and the reverse: stream order is what keeps updated values out of the gradients.  No float atomics anywhere,
// so a step is a pure function of its inputs.

#include "common.cuh"

namespace lk {

constexpr int FLEXMF_UNIT = 64;

__host__ __device__ __forceinline__ uint64_t flexmf_mix(uint64_t x)
{
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}

// the draw of (seed, step, pos, rep, attempt) in [0, n): see lk_flexmf_sample_negatives in the header
__device__ __forceinline__ uint32_t flexmf_draw(uint64_t seed, uint64_t step, uint64_t pos, uint64_t rep,
                                                uint64_t attempt, uint64_t n)
{
    const uint64_t g = 0x9e3779b97f4a7c15ull;
    uint64_t h = flexmf_mix(seed + g * (step + 1));
    h = flexmf_mix(h + g * (pos + 1));
    h = flexmf_mix(h + g * ((rep << 32) + attempt + 1));
    return static_cast<uint32_t>(((h >> 32) * n) >> 32);
}

__global__ void flexmf_sample_kernel(lk_flexmf_sample_args a)
{
    int64_t t = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (t >= a.n_samples * a.n) return;
    int64_t g = t / a.n;
    int rep = int(t - g * a.n);
    int64_t step = a.step0 + g / a.batch_size;
    int64_t pos = g % a.batch_size;
    int row = a.d_rows[g];
    const int32_t *cols = a.d_ui_cols;
    int lo0 = a.d_ui_indptr[row], hi0 = a.d_ui_indptr[row + 1];
    int c = 0;
    for (int attempt = 0;; ++attempt) {
        if (a.popular)
            c = a.d_coo_items[flexmf_draw(a.seed, step, pos, rep, attempt, uint64_t(a.nnz))];
        else
            c = int(flexmf_draw(a.seed, step, pos, rep, attempt, uint64_t(a.n_items)));
        if (attempt >= a.max_attempts) break;
        int lo = lo0, hi = hi0;  // first column >= c
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (cols[mid] < c)
                lo = mid + 1;
            else
                hi = mid;
        }
        if (lo == hi0 || cols[lo] != c) break;
    }
    a.d_out[t] = c;
}

// ---------------------------------------------------------------------------------------------------------------
// a parameter row across one warp: 4 floats per lane.  V4 (k % 4 == 0): lane l holds columns 4l..4l+3 as one float4
// load (k = 64 leaves the upper half-warp without columns: accepted, the gathers are still whole 256 B rows);
// otherwise lane l holds columns l, l+32, l+64, l+96.
// ---------------------------------------------------------------------------------------------------------------
template <bool V4>
__device__ __forceinline__ void load_row(float (&v)[4], const float *row, int k, int lane)
{
    if (V4) {
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (lane * 4 < k) x = *reinterpret_cast<const float4 *>(row + lane * 4);
        v[0] = x.x, v[1] = x.y, v[2] = x.z, v[3] = x.w;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = lane + 32 * j < k ? row[lane + 32 * j] : 0.f;
    }
}

template <bool V4>
__device__ __forceinline__ void store_row(const float (&v)[4], float *row, int k, int lane)
{
    if (V4) {
        if (lane * 4 < k) *reinterpret_cast<float4 *>(row + lane * 4) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (lane + 32 * j < k) row[lane + 32 * j] = v[j];
    }
}

__device__ __forceinline__ float dot4(const float (&a)[4], const float (&b)[4])
{
    return warp_sum(fmaf(a[3], b[3], fmaf(a[2], b[2], fmaf(a[1], b[1], a[0] * b[0]))));
}

// log(1 + e^x) and 1 / (1 + e^-x) without overflow
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x)
{
    float e = expf(-fabsf(x));
    return (x >= 0.f ? 1.f : e) / (1.f + e);
}

template <bool V4>
__global__ void __launch_bounds__(256) flexmf_forward_kernel(lk_flexmf_step_args a, float *coef, float *sample_loss)
{
    int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= a.batch) return;
    const int n = a.n_neg, k = a.k;
    const bool mse = a.loss == LK_FLEXMF_MSE;
    const bool l2 = a.reg_method == LK_FLEXMF_REG_L2 && !mse;  // the MSE loss reported is without the norm term
    int u = a.d_users[w];
    float uv[4], iv[4];
    load_row<V4>(uv, a.d_u_emb + int64_t(u) * k, k, lane);
    float ub = a.d_u_bias ? a.d_u_bias[u] : 0.f;
    float nu = l2 ? sqrtf(dot4(uv, uv)) : 0.f;
    float inv_pos = 1.f / float(a.batch), inv_neg = n > 0 ? 1.f / (float(a.batch) * float(n)) : 0.f;
    float inv_all = 1.f / (float(a.batch) + float(a.batch) * float(n));
    float loss = 0.f, s_pos = 0.f, c_pos = 0.f;
    for (int j = 0; j <= n; ++j) {
        int it = j == 0 ? a.d_pos[w] : a.d_neg[int64_t(w) * n + j - 1];
        load_row<V4>(iv, a.d_i_emb + int64_t(it) * k, k, lane);
        float ib = a.d_i_bias ? a.d_i_bias[it] : 0.f;
        float s = ub + ib + dot4(uv, iv);
        if (l2) {
            float nrm = ub * ub + ib * ib + nu + sqrtf(dot4(iv, iv));
            loss += a.regularization * 0.5f * nrm * (j == 0 ? inv_pos : inv_neg);
        }
        float c;
        if (mse) {  // n = 0: the rating's target t = r - mu
            float d = s - a.d_ratings[w];
            loss = d * d * inv_pos;
            c = 2.f * d * inv_pos;
        } else if (a.loss == LK_FLEXMF_LOGISTIC) {
            if (j == 0) {
                loss += a.positive_weight * softplus(-s) * inv_all;
                c = -a.positive_weight * sigmoid(-s) * inv_all;
            } else {
                loss += softplus(s) * inv_all;
                c = sigmoid(s) * inv_all;
            }
        } else {
            if (j == 0) {
                s_pos = s;
                continue;  // the positive's coefficient is minus the sum of its pairs'
            }
            float d = s_pos - s;
            loss += softplus(-d) * inv_neg;
            c = sigmoid(-d) * inv_neg;
            c_pos -= c;
        }
        if (lane == 0) coef[int64_t(w) * (n + 1) + j] = c;
    }
    if (lane == 0) {
        if (a.loss == LK_FLEXMF_PAIRWISE) coef[int64_t(w) * (n + 1)] = c_pos;
        sample_loss[w] = loss;
    }
}

__global__ void __launch_bounds__(1024) flexmf_loss_kernel(const float *sample_loss, int batch, float *out)
{
    __shared__ double part[1024];
    double s = 0.0;
    for (int i = threadIdx.x; i < batch; i += 1024) s += double(sample_loss[i]);
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if (int(threadIdx.x) < o) part[threadIdx.x] += part[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = float(part[0]);
}

// partials: [unit][kp] floats, the embedding gradient in columns 0..k-1 and the bias gradient in column k
__host__ __device__ __forceinline__ int flexmf_kp(int k) { return (k + 1 + 3) & ~3; }

template <bool V4>
__global__ void flexmf_grad_kernel(lk_flexmf_step_args a, const float *coef, float *partials)
{
    int x = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (x >= a.n_u_units + a.n_i_units) return;
    const int n = a.n_neg, k = a.k, kp = flexmf_kp(k);
    const bool l2 = a.reg_method == LK_FLEXMF_REG_L2;
    const bool user_side = x < a.n_u_units;
    const lk_flexmf_groups &g = user_side ? a.u_groups : a.i_groups;
    const int64_t unit = (user_side ? x : x - a.n_u_units) + g.unit0;
    // the item rows' L2 weight per occurrence, over regularization / B: 1/2 for the implicit positive (half of
    // reg/2 (mean norm+ + mean norm-)), 1 for MSE (reg mean norm)
    const float i_l2 = a.loss == LK_FLEXMF_MSE ? 1.f : 0.5f;
    const int32_t uniq = g.d_unit_uniq[unit];
    const int row = g.d_uniq_row[uniq];
    const int64_t p0 = g.d_unit_start[unit], p1 = g.d_unit_start[unit + 1];
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, accb = 0.f, ov[4];
    const float inv_pos = 1.f / float(a.batch), inv_neg = n > 0 ? 1.f / (float(a.batch) * float(n)) : 0.f;
    if (user_side) {
        for (int64_t p = p0; p < p1; ++p) {
            int b = g.d_occ[p];
            float t[4] = {0.f, 0.f, 0.f, 0.f}, tb = 0.f;  // the sample's items are combined first
            for (int j = 0; j <= n; ++j) {
                int it = j == 0 ? a.d_pos[b] : a.d_neg[int64_t(b) * n + j - 1];
                float c = coef[int64_t(b) * (n + 1) + j];
                load_row<V4>(ov, a.d_i_emb + int64_t(it) * k, k, lane);
#pragma unroll
                for (int q = 0; q < 4; ++q) t[q] = fmaf(c, ov[q], t[q]);
                tb += c;
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] += t[q];
            // the user bias cancels in s+ - s-: its pairwise gradient is exactly 0, not the rounding residue of
            // c_pos + sum(c_r)
            if (a.loss != LK_FLEXMF_PAIRWISE) accb += tb;
        }
        // d/du of reg/2 (mean(norm+) + mean(norm-)): the user is in the positive and in all n negatives; of MSE's
        // reg mean(norm): once per sample.  Either way reg/B per occurrence
        if (l2) {
            float cnt = float(p1 - p0);
            load_row<V4>(ov, a.d_u_emb + int64_t(row) * k, k, lane);
            float nrm = sqrtf(dot4(ov, ov));
            float wv = nrm > 0.f ? cnt * a.regularization * inv_pos / nrm : 0.f;  // d|x|/dx at 0 is 0, as in torch
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(wv, ov[q], acc[q]);
            if (a.d_u_bias) accb = fmaf(cnt * 2.f * a.regularization * inv_pos, a.d_u_bias[row], accb);
        }
    } else {
        float wl2 = 0.f;
        for (int64_t p = p0; p < p1; ++p) {
            int slot = g.d_occ[p];
            int b = slot / (n + 1);
            float c = coef[slot];
            load_row<V4>(ov, a.d_u_emb + int64_t(a.d_users[b]) * k, k, lane);
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(c, ov[q], acc[q]);
            accb += c;
            wl2 += slot - b * (n + 1) == 0 ? inv_pos : inv_neg;
        }
        if (l2) {
            load_row<V4>(ov, a.d_i_emb + int64_t(row) * k, k, lane);
            float nrm = sqrtf(dot4(ov, ov));
            float wv = nrm > 0.f ? i_l2 * a.regularization * wl2 / nrm : 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(wv, ov[q], acc[q]);
            if (a.d_i_bias) accb = fmaf(2.f * i_l2 * a.regularization * wl2, a.d_i_bias[row], accb);
        }
    }
    float *out = partials + int64_t(x) * kp;
    store_row<V4>(acc, out, k, lane);
    if (lane == 0) {
        out[k] = accb;
        // AdamW sweeps every row: the first unit of a row tells the sweep where the row's partials are
        if (g.d_mark != nullptr && unit == g.d_uniq_unit[uniq]) g.d_mark[row] = (a.step << 32) | int64_t(uniq);
    }
}

struct FlexmfTable {
    float *w, *m, *v;   // parameters and the two moments, [n_rows][k]
    int k, col0;        // col0: the table's first column in a partials row
    int64_t n_threads;  // dense: n_rows * k / W; sparse: n_uniq * k / W
    int64_t block0;     // first block of the grid that works on this table
    int side;           // 0 users, 1 items
};
struct FlexmfTables {
    FlexmfTable t[4];
};

template <int W>
__device__ __forceinline__ void flexmf_adam(const lk_flexmf_step_args &a, const FlexmfTable &tab, int64_t t,
                                            const float *partials)
{
    const bool dense = a.reg_method == LK_FLEXMF_REG_ADAMW;
    const lk_flexmf_groups &g = tab.side == 0 ? a.u_groups : a.i_groups;
    const int kp = flexmf_kp(a.k);
    int64_t e = t * W;
    int64_t r = e / tab.k;
    int col = int(e - r * tab.k);
    int64_t row, uniq = -1;
    if (dense) {
        row = r;
        int64_t mk = g.d_mark[row];
        if ((mk >> 32) == a.step) uniq = mk & 0xffffffffll;
    } else {
        uniq = g.uniq0 + r;
        row = g.d_uniq_row[uniq];
    }
    float grad[W];
#pragma unroll
    for (int q = 0; q < W; ++q) grad[q] = 0.f;
    if (uniq >= 0) {  // the row's units, in order
        const int64_t local0 = g.unit0 - (tab.side == 0 ? 0 : a.n_u_units);
        for (int64_t unit = g.d_uniq_unit[uniq]; unit < g.d_uniq_unit[uniq + 1]; ++unit) {
            const float *p = partials + (unit - local0) * kp + tab.col0 + col;
            if constexpr (W == 4) {
                float4 x = *reinterpret_cast<const float4 *>(p);
                grad[0] += x.x, grad[1] += x.y, grad[2] += x.z, grad[3] += x.w;
            } else {
                grad[0] += p[0];
            }
        }
    }
    float pw[W], pm[W], pv[W];
    const int64_t at = row * tab.k + col;
    if constexpr (W == 4) {
        float4 x = *reinterpret_cast<const float4 *>(tab.w + at);
        float4 y = *reinterpret_cast<const float4 *>(tab.m + at);
        float4 z = *reinterpret_cast<const float4 *>(tab.v + at);
        pw[0] = x.x, pw[1] = x.y, pw[2] = x.z, pw[3] = x.w;
        pm[0] = y.x, pm[1] = y.y, pm[2] = y.z, pm[3] = y.w;
        pv[0] = z.x, pv[1] = z.y, pv[2] = z.z, pv[3] = z.w;
    } else {
        pw[0] = tab.w[at], pm[0] = tab.m[at], pv[0] = tab.v[at];
    }
#pragma unroll
    for (int q = 0; q < W; ++q) {
        float gr = grad[q];
        if (dense) {  // torch.optim.AdamW: decoupled decay, then Adam with eps added after the bias correction
            pw[q] *= a.decay;
            pm[q] = fmaf(gr - pm[q], a.one_minus_beta1, pm[q]);
            pv[q] = fmaf(a.one_minus_beta2 * gr, gr, pv[q] * a.beta2);
            float denom = sqrtf(pv[q]) / a.bias2_sqrt + a.eps;
            pw[q] = fmaf(-a.step_size, pm[q] / denom, pw[q]);
        } else {  // torch.optim.SparseAdam: eps added before the bias correction, which is folded into step_size
            pm[q] += (gr - pm[q]) * a.one_minus_beta1;
            pv[q] += (gr * gr - pv[q]) * a.one_minus_beta2;
            pw[q] = fmaf(-a.step_size, pm[q] / (sqrtf(pv[q]) + a.eps), pw[q]);
        }
    }
    if constexpr (W == 4) {
        *reinterpret_cast<float4 *>(tab.w + at) = make_float4(pw[0], pw[1], pw[2], pw[3]);
        *reinterpret_cast<float4 *>(tab.m + at) = make_float4(pm[0], pm[1], pm[2], pm[3]);
        *reinterpret_cast<float4 *>(tab.v + at) = make_float4(pv[0], pv[1], pv[2], pv[3]);
    } else {
        tab.w[at] = pw[0], tab.m[at] = pm[0], tab.v[at] = pv[0];
    }
}

template <bool V4>
__global__ void __launch_bounds__(256)
    flexmf_update_kernel(lk_flexmf_step_args a, FlexmfTables tabs, const float *partials)
{
    int ti = 3;
    while (ti > 0 && int64_t(blockIdx.x) < tabs.t[ti].block0) --ti;
    const FlexmfTable &tab = tabs.t[ti];
    int64_t t = (int64_t(blockIdx.x) - tab.block0) * blockDim.x + threadIdx.x;
    if (t >= tab.n_threads) return;
    if (V4 && tab.k > 1)
        flexmf_adam<4>(a, tab, t, partials);
    else
        flexmf_adam<1>(a, tab, t, partials);
}

static int64_t flexmf_max_units(int64_t occurrences)
{
    return occurrences + occurrences / FLEXMF_UNIT + 1;
}

static int64_t flexmf_ws_bytes(int64_t batch, int64_t n_neg, int k)
{
    int64_t units = flexmf_max_units(batch) + flexmf_max_units(batch * (n_neg + 1));
    return 4 * (units * flexmf_kp(k) + batch * (n_neg + 1) + batch);  // partials, coef, sample_loss
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_flexmf_sample_negatives(const lk_flexmf_sample_args *a, void *stream)
{
    LK_REQUIRE(a != nullptr, LK_ERR_INVALID, "lk_flexmf_sample_negatives: null arguments");
    LK_REQUIRE(a->n_users > 0 && a->n_items > 0 && a->n >= 1 && a->batch_size >= 1 && a->n_samples >= 0,
               LK_ERR_INVALID, "lk_flexmf_sample_negatives: n_users, n_items, n and batch_size must be positive");
    LK_REQUIRE(a->max_attempts >= 0 && a->step0 >= 0, LK_ERR_INVALID,
               "lk_flexmf_sample_negatives: max_attempts and step0 must not be negative");
    LK_REQUIRE(!a->popular || (a->d_coo_items != nullptr && a->nnz > 0 && a->nnz < (int64_t(1) << 32)),
               LK_ERR_INVALID, "lk_flexmf_sample_negatives: popular sampling needs the COO items, 0 < nnz < 2^32");
    LK_REQUIRE(a->d_ui_indptr && a->d_ui_cols && a->d_rows && a->d_out, LK_ERR_INVALID,
               "lk_flexmf_sample_negatives: null device pointer");
    int64_t threads = a->n_samples * a->n;
    if (threads == 0) return LK_OK;
    LK_REQUIRE((threads + 255) / 256 < (int64_t(1) << 31), LK_ERR_UNSUPPORTED,
               "lk_flexmf_sample_negatives: n_samples * n is too large for one launch");
    flexmf_sample_kernel<<<unsigned((threads + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(*a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_flexmf_workspace_bytes(int32_t batch, int32_t n_neg, int32_t k, int64_t *bytes)
{
    LK_REQUIRE(bytes != nullptr, LK_ERR_INVALID, "lk_flexmf_workspace_bytes: null result pointer");
    LK_REQUIRE(batch >= 1 && n_neg >= 0, LK_ERR_INVALID,
               "lk_flexmf_workspace_bytes: batch must be positive and n_neg not negative");
    LK_REQUIRE(k >= 1 && k <= lk_als_max_features(), LK_ERR_UNSUPPORTED,
               "lk_flexmf_workspace_bytes: k=%d is outside 1..%d", k, lk_als_max_features());
    LK_REQUIRE(int64_t(batch) * (n_neg + 1) < (int64_t(1) << 30), LK_ERR_UNSUPPORTED,
               "lk_flexmf_workspace_bytes: batch * (n_neg + 1) must be below 2^30");
    *bytes = flexmf_ws_bytes(batch, n_neg, k);
    return LK_OK;
}

int lk_flexmf_step(const lk_flexmf_step_args *a, void *stream)
{
    LK_REQUIRE(a != nullptr, LK_ERR_INVALID, "lk_flexmf_step: null arguments");
    int64_t need = 0;
    int rc = lk_flexmf_workspace_bytes(a->batch, a->n_neg, a->k, &need);
    if (rc != LK_OK) return rc;
    LK_REQUIRE(a->d_workspace != nullptr && a->workspace_bytes >= need, LK_ERR_INVALID,
               "lk_flexmf_step: the workspace has %lld bytes, the step needs %lld", (long long)a->workspace_bytes,
               (long long)need);
    LK_REQUIRE(a->loss == LK_FLEXMF_LOGISTIC || a->loss == LK_FLEXMF_PAIRWISE || a->loss == LK_FLEXMF_MSE,
               LK_ERR_INVALID, "lk_flexmf_step: unknown loss %d", a->loss);
    const bool mse = a->loss == LK_FLEXMF_MSE;
    LK_REQUIRE(mse == (a->n_neg == 0), LK_ERR_INVALID,
               "lk_flexmf_step: MSE takes no negatives (n_neg = 0); the other losses take n_neg >= 1 (n_neg = %d)",
               a->n_neg);
    LK_REQUIRE(!mse || a->d_ratings != nullptr, LK_ERR_INVALID, "lk_flexmf_step: MSE needs the targets d_ratings");
    LK_REQUIRE(a->reg_method >= LK_FLEXMF_REG_NONE && a->reg_method <= LK_FLEXMF_REG_ADAMW, LK_ERR_INVALID,
               "lk_flexmf_step: unknown reg_method %d", a->reg_method);
    LK_REQUIRE(a->step >= 1 && a->step < (int64_t(1) << 31) && a->n_users > 0 && a->n_items > 0, LK_ERR_INVALID,
               "lk_flexmf_step: step counts from 1 and stays below 2^31; n_users and n_items must be positive");
    const bool dense = a->reg_method == LK_FLEXMF_REG_ADAMW;
    LK_REQUIRE(!dense || (a->u_groups.d_mark && a->i_groups.d_mark), LK_ERR_INVALID,
               "lk_flexmf_step: AdamW needs the row marks of both sides");
    LK_REQUIRE(a->n_u_units >= 1 && a->n_u_units <= flexmf_max_units(a->batch) && a->n_i_units >= 1 &&
                   a->n_i_units <= flexmf_max_units(int64_t(a->batch) * (a->n_neg + 1)),
               LK_ERR_INVALID, "lk_flexmf_step: unit counts outside what the workspace holds");
    LK_REQUIRE(a->u_groups.n_uniq >= 1 && a->u_groups.n_uniq <= a->n_u_units && a->i_groups.n_uniq >= 1 &&
                   a->i_groups.n_uniq <= a->n_i_units,
               LK_ERR_INVALID, "lk_flexmf_step: a side has more rows than units");
    LK_REQUIRE(a->d_u_emb && a->d_u_emb_m && a->d_u_emb_v && a->d_i_emb && a->d_i_emb_m && a->d_i_emb_v &&
                   a->d_users && a->d_pos && (a->d_neg || mse) && a->d_loss,
               LK_ERR_INVALID, "lk_flexmf_step: null device pointer");
    LK_REQUIRE((a->d_u_bias == nullptr) == (a->d_u_bias_m == nullptr) &&
                   (a->d_u_bias == nullptr) == (a->d_u_bias_v == nullptr) &&
                   (a->d_i_bias == nullptr) == (a->d_i_bias_m == nullptr) &&
                   (a->d_i_bias == nullptr) == (a->d_i_bias_v == nullptr),
               LK_ERR_INVALID, "lk_flexmf_step: a bias vector and its two moments go together");

    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int k = a->k, B = a->batch;
    float *partials = static_cast<float *>(a->d_workspace);  // first: its rows are read as float4
    float *coef = partials + (flexmf_max_units(B) + flexmf_max_units(int64_t(B) * (a->n_neg + 1))) * flexmf_kp(k);
    float *sample_loss = coef + int64_t(B) * (a->n_neg + 1);
    const bool v4 = k % 4 == 0;
    const unsigned fwd_blocks = unsigned((int64_t(B) * 32 + 255) / 256);
    const unsigned grad_blocks = unsigned(((int64_t(a->n_u_units) + a->n_i_units) * 32 + 255) / 256);

    FlexmfTables tabs;
    int64_t block = 0;
    auto table = [&](int idx, float *w, float *m, float *v, int tk, int col0, int side) {
        FlexmfTable &t = tabs.t[idx];
        int64_t rows = dense ? (side == 0 ? a->n_users : a->n_items)
                             : (side == 0 ? a->u_groups.n_uniq : a->i_groups.n_uniq);
        t = FlexmfTable{w, m, v, tk, col0, w ? rows * tk / ((v4 && tk > 1) ? 4 : 1) : 0, block, side};
        block += (t.n_threads + 255) / 256;
    };
    table(0, a->d_u_emb, a->d_u_emb_m, a->d_u_emb_v, k, 0, 0);
    table(1, a->d_i_emb, a->d_i_emb_m, a->d_i_emb_v, k, 0, 1);
    table(2, a->d_u_bias, a->d_u_bias_m, a->d_u_bias_v, 1, k, 0);
    table(3, a->d_i_bias, a->d_i_bias_m, a->d_i_bias_v, 1, k, 1);
    LK_REQUIRE(block < (int64_t(1) << 31), LK_ERR_UNSUPPORTED, "lk_flexmf_step: the tables are too large for one launch");

    if (v4) {
        flexmf_forward_kernel<true><<<fwd_blocks, 256, 0, s>>>(*a, coef, sample_loss);
        flexmf_loss_kernel<<<1, 1024, 0, s>>>(sample_loss, B, a->d_loss);
        flexmf_grad_kernel<true><<<grad_blocks, 256, 0, s>>>(*a, coef, partials);
        flexmf_update_kernel<true><<<unsigned(block), 256, 0, s>>>(*a, tabs, partials);
    } else {
        flexmf_forward_kernel<false><<<fwd_blocks, 256, 0, s>>>(*a, coef, sample_loss);
        flexmf_loss_kernel<<<1, 1024, 0, s>>>(sample_loss, B, a->d_loss);
        flexmf_grad_kernel<false><<<grad_blocks, 256, 0, s>>>(*a, coef, partials);
        flexmf_update_kernel<false><<<unsigned(block), 256, 0, s>>>(*a, tabs, partials);
    }
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
