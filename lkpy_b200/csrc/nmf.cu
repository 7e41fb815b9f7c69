// nmf.cu — scikit-learn's NMF coordinate descent (solver="cd", NMFScorer) for sm_90a, bit for bit.
//
// lk_nmf_cd_sweep is one `_update_cdnmf_fast(W, HHt, XHt, arange(k))` call (sklearn/decomposition/_cdnmf_fast.pyx):
//     for t in 0..k-1:  for i in 0..n-1:
//         grad = -XHt[i][t];  for r in 0..k-1: grad = grad + HHt[t][r] * W[i][r]
//         pg = W[i][t] == 0 ? min(0, grad) : grad;   violation += |pg|
//         if HHt[t][t] != 0: W[i][t] = max(W[i][t] - grad / HHt[t][t], 0)
// Within one component t the rows are independent, and row i reads only its own W row, so a thread owns a row for
// all k components and the (t, i) order only matters for the violation.  The sweep writes every |pg| to a [k][n]
// buffer in t-major order instead, and lk_f32_seq_sum adds them up in that order.  Products, sums and the quotient
// are __fmul_rn / __fadd_rn / __fdiv_rn, so nothing is contracted to an FFMA.  HHt and the CTA's W rows live in
// shared memory; the W rows are stored column by column with the thread index fastest, so that lanes never share a
// bank.
//
// lk_f32_seq_sum is the left-to-right f32 sum s = fl(s + x[j]) from s = +0 of n non-negative values.  While s stays
// in one binade with ulp u (the subnormals and the first normal binade together form one with u = 2^-149), every
// step is s <- s + rne(x[j] / u) u, an integer count of ulps whose only dependence on s is the parity of s / u when
// x[j] / u is an exact tie.  So each element is a map from that parity to (increment, new parity), maps compose, and a
// block-wide scan of maps gives every partial sum of the binade exactly.  The first element whose partial sum would
// leave the binade is added with __fadd_rn instead, and the walk restarts after it in the new binade.  s only
// grows, so there is one restart per binade crossed (a few dozen for violations), plus one per inf or NaN.
#include <algorithm>

#include "common.cuh"

namespace lk {

constexpr int NMF_SWEEP_CT = 128;  // rows per CTA

__global__ void __launch_bounds__(NMF_SWEEP_CT) nmf_cd_sweep_kernel(const lk_nmf_cd_sweep_args a)
{
    extern __shared__ float nmf_smem[];
    const int k = a.k;
    float *hh = nmf_smem;                                  // HHt [k][k]
    float *wi = nmf_smem + k * k + threadIdx.x;            // this row's W[r] at wi[r * NMF_SWEEP_CT]
    for (int e = threadIdx.x; e < k * k; e += NMF_SWEEP_CT) hh[e] = __ldg(a.d_hht + e);
    const int i = blockIdx.x * NMF_SWEEP_CT + threadIdx.x;
    const bool on = i < a.n;
    if (on)
        for (int r = 0; r < k; r++) wi[r * NMF_SWEEP_CT] = a.d_w[(int64_t)i * k + r];
    __syncthreads();
    if (!on) return;
    const float *xi = a.d_xht + (int64_t)i * k;
    for (int t = 0; t < k; t++) {
        const float *ht = hh + t * k;
        float grad = -__ldg(xi + t);
        for (int r = 0; r < k; r++) grad = __fadd_rn(grad, __fmul_rn(ht[r], wi[r * NMF_SWEEP_CT]));
        const float w = wi[t * NMF_SWEEP_CT];
        // Cython's min(0., grad) and max(v, 0.) keep their first argument unless the second compares less/greater
        const float pg = w == 0.0f ? (grad < 0.0f ? grad : 0.0f) : grad;
        a.d_pg[(int64_t)t * a.n + i] = fabsf(pg);
        const float hess = ht[t];
        if (hess != 0.0f) {
            const float v = __fsub_rn(w, __fdiv_rn(grad, hess));
            wi[t * NMF_SWEEP_CT] = 0.0f > v ? 0.0f : v;
        }
    }
    for (int r = 0; r < k; r++) a.d_w[(int64_t)i * k + r] = wi[r * NMF_SWEEP_CT];
}

// ---- lk_f32_seq_sum ------------------------------------------------------------------------------------------------

constexpr int SEQ_CT = 512;
constexpr int SEQ_ITEMS = 16;                       // consecutive elements per thread
constexpr int SEQ_TILE = SEQ_CT * SEQ_ITEMS;
constexpr long long SEQ_LIMIT = 1LL << 24;          // ulps in a binade: s / u < 2^24 inside it
constexpr long long SEQ_BIG = 1LL << 26;            // any increment this large leaves the binade

constexpr int SEQ_MAX_SUMS = 8;  // sums per lk_f32_seq_sum call, one CTA each

struct SeqSumBatch {
    lk_f32_seq_sum_args sums[SEQ_MAX_SUMS];
};

// parity -> (increment in ulps, parity after); out holds the two parities after as bits 0 (from even) and 1 (from odd)
struct SeqMap {
    long long inc0, inc1;
    int out;
};

__device__ __forceinline__ SeqMap seq_identity() { return {0, 0, 0b10}; }

// a, then b
__device__ __forceinline__ SeqMap seq_compose(const SeqMap &a, const SeqMap &b)
{
    const int a0 = a.out & 1, a1 = a.out >> 1;
    return {a.inc0 + (a0 ? b.inc1 : b.inc0), a.inc1 + (a1 ? b.inc1 : b.inc0),
            ((b.out >> a0) & 1) | (((b.out >> a1) & 1) << 1)};
}

// the map of adding x in the binade whose ulp is 2^ue
__device__ __forceinline__ SeqMap seq_element(float x, int ue)
{
    const unsigned b = __float_as_uint(x) & 0x7fffffffu;
    const int ex = (int)(b >> 23);
    if (ex == 0xff) return {SEQ_BIG, SEQ_BIG, 0b10};  // inf or NaN: leaves the binade, added by __fadd_rn
    const long long m = ex == 0 ? (long long)(b & 0x7fffff) : (long long)((b & 0x7fffff) | 0x800000);
    const int sh = ue - (ex == 0 ? -149 : ex - 150);  // x / u = m / 2^sh
    long long r;
    if (sh <= 0) {
        r = -sh >= 26 ? SEQ_BIG : min(m << -sh, SEQ_BIG);
    } else {
        const int s = sh > 26 ? 26 : sh;  // m < 2^24 <= half from here on: rounds to 0
        const long long f = m >> s, rem = m & ((1LL << s) - 1), half = 1LL << (s - 1);
        if (rem == half) {  // a tie: to the even count, which leaves the parity even
            return {f + (f & 1), f + ((f + 1) & 1), 0b00};
        }
        r = f + (rem > half);
    }
    const int o = (int)(r & 1);
    return {r, r, o | ((1 ^ o) << 1)};
}

struct SeqSegment {
    int ue;          // log2 of the ulp
    long long cnt;   // s / u
};

__device__ __forceinline__ SeqSegment seq_segment(float s)
{
    const unsigned b = __float_as_uint(s);
    const int ex = (int)(b >> 23);
    if (ex <= 1) return {-149, (long long)b};
    return {ex - 150, (long long)((b & 0x7fffff) | 0x800000)};
}

__device__ __forceinline__ float seq_value(int ue, long long cnt)
{
    if (ue == -149) return __uint_as_float((unsigned)cnt);
    return __uint_as_float(((unsigned)(ue + 150) << 23) | ((unsigned)cnt & 0x7fffff));
}

__device__ __forceinline__ SeqMap shfl_up_map(const SeqMap &m, int d)
{
    return {(long long)__shfl_up_sync(FULL, (unsigned long long)m.inc0, d),
            (long long)__shfl_up_sync(FULL, (unsigned long long)m.inc1, d), __shfl_up_sync(FULL, m.out, d)};
}

__global__ void __launch_bounds__(SEQ_CT) f32_seq_sum_kernel(const SeqSumBatch batch)
{
    const lk_f32_seq_sum_args a = batch.sums[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ SeqMap warp_maps[SEQ_CT / 32];
    __shared__ long long sh_pos, sh_cross, sh_cnt_before;
    __shared__ int sh_ue, sh_mode;  // mode 0: finite; 1: s is +inf; 2: s is NaN
    __shared__ long long sh_end_cnt;
    __shared__ float sh_s;
    if (tid == 0) {
        sh_pos = 0;
        sh_ue = -149;
        sh_mode = 0;
        sh_s = 0.0f;
    }
    __syncthreads();
    const long long n = a.n;
    while (true) {
        const long long pos = sh_pos;
        const int mode = sh_mode;
        if (pos >= n || mode == 2) break;
        const long long base = pos + (long long)tid * SEQ_ITEMS;
        float x[SEQ_ITEMS];
#pragma unroll
        for (int q = 0; q < SEQ_ITEMS; q++) x[q] = base + q < n ? __ldg(a.d_x + base + q) : 0.0f;
        if (mode == 1) {  // inf + finite stays inf; only a NaN changes it
            bool nan = false;
#pragma unroll
            for (int q = 0; q < SEQ_ITEMS; q++) nan |= x[q] != x[q];
            const int any = __syncthreads_or(nan);
            if (tid == 0) {
                if (any) sh_mode = 2, sh_s = __int_as_float(0x7fc00000);
                sh_pos = pos + SEQ_TILE;
            }
            __syncthreads();
            continue;
        }
        const int ue = sh_ue;
        const long long cnt0 = seq_segment(sh_s).cnt;
        const int par0 = (int)(cnt0 & 1);
        SeqMap mine = seq_identity();
#pragma unroll
        for (int q = 0; q < SEQ_ITEMS; q++) mine = seq_compose(mine, seq_element(x[q], ue));
        // inclusive warp scan, then the warps' totals, then this thread's exclusive prefix
        SeqMap incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const SeqMap o = shfl_up_map(incl, d);
            if (lane >= d) incl = seq_compose(o, incl);
        }
        if (lane == 31) warp_maps[warp] = incl;
        if (tid == 0) sh_cross = n;
        __syncthreads();
        SeqMap pre = seq_identity();
        for (int w = 0; w < warp; w++) pre = seq_compose(pre, warp_maps[w]);
        SeqMap ex = shfl_up_map(incl, 1);
        if (lane == 0) ex = seq_identity();
        pre = seq_compose(pre, ex);
        long long cnt = cnt0 + (par0 ? pre.inc1 : pre.inc0);
        int par = (pre.out >> par0) & 1;
        long long cross = n, cnt_before = 0;
#pragma unroll
        for (int q = 0; q < SEQ_ITEMS; q++) {
            if (cross == n && base + q < n) {
                const SeqMap e = seq_element(x[q], ue);
                const long long c = cnt + (par ? e.inc1 : e.inc0);
                if (c >= SEQ_LIMIT) {
                    cross = base + q, cnt_before = cnt;
                } else {
                    cnt = c;
                    par = (e.out >> par) & 1;
                }
            }
        }
        if (cross < n) atomicMin((unsigned long long *)&sh_cross, (unsigned long long)cross);
        if (tid == SEQ_CT - 1) sh_end_cnt = cnt;
        __syncthreads();
        if (cross < n && cross == sh_cross) sh_cnt_before = cnt_before;
        __syncthreads();
        if (tid == 0) {
            if (sh_cross < n) {
                const float s = __fadd_rn(seq_value(ue, sh_cnt_before), __ldg(a.d_x + sh_cross));
                if (s != s) {
                    sh_mode = 2;
                } else if (isinf(s)) {
                    sh_mode = 1;
                } else {
                    sh_ue = seq_segment(s).ue;
                }
                sh_s = s;
                sh_pos = sh_cross + 1;
            } else {
                sh_s = seq_value(ue, sh_end_cnt);
                sh_pos = pos + SEQ_TILE;
            }
        }
        __syncthreads();
    }
    if (tid == 0) *a.d_out = sh_s;
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_nmf_cd_sweep(const lk_nmf_cd_sweep_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_nmf_cd_sweep: null args");
    const lk_nmf_cd_sweep_args &a = *args;
    LK_REQUIRE(a.n >= 0, LK_ERR_INVALID, "lk_nmf_cd_sweep: n must be non-negative");
    LK_REQUIRE(a.k >= 1 && a.k <= 128, LK_ERR_UNSUPPORTED, "lk_nmf_cd_sweep: k must be in 1..128");
    if (a.n == 0) return LK_OK;
    LK_REQUIRE(a.d_w && a.d_hht && a.d_xht && a.d_pg, LK_ERR_INVALID, "lk_nmf_cd_sweep: null input or output");
    const size_t smem = sizeof(float) * ((size_t)a.k * a.k + (size_t)a.k * NMF_SWEEP_CT);
    LK_CUDA_TRY(cudaFuncSetAttribute(nmf_cd_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned grid = (unsigned)((a.n + NMF_SWEEP_CT - 1) / NMF_SWEEP_CT);
    nmf_cd_sweep_kernel<<<grid, NMF_SWEEP_CT, smem, static_cast<cudaStream_t>(stream)>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

int lk_f32_seq_sum(const lk_f32_seq_sum_args *sums, int32_t count, void *stream)
{
    LK_REQUIRE(sums != nullptr, LK_ERR_INVALID, "lk_f32_seq_sum: null args");
    LK_REQUIRE(count >= 1 && count <= SEQ_MAX_SUMS, LK_ERR_INVALID, "lk_f32_seq_sum: count must be in 1..8");
    SeqSumBatch batch{};
    for (int i = 0; i < count; i++) {
        LK_REQUIRE(sums[i].n >= 0 && sums[i].d_out && (sums[i].n == 0 || sums[i].d_x), LK_ERR_INVALID,
                   "lk_f32_seq_sum: n must be non-negative, and the input and output non-null");
        batch.sums[i] = sums[i];
    }
    f32_seq_sum_kernel<<<(unsigned)count, SEQ_CT, 0, static_cast<cudaStream_t>(stream)>>>(batch);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
