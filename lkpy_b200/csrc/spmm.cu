// spmm.cu — sparse (CSR) x dense products for sm_90a, bit for bit with SciPy's f32 `A @ D`, `A.T @ D` and `D.T @ A`.
//
// Y [n_rows][W] = A x D, D [n_src][W] row-major.  For every output element (row r, column c):
//     acc = +0.0f;  for p in A's row r in stored order: acc = acc + (val[p] * D[idx[p]][c])    (each op rounded)
// which is what SciPy's csr_matvecs computes for `A @ D`.  `A.T @ D` (csc_matvecs, a scatter over A's rows) adds
// into output row j in ascending row order, which is this walk over the transposed CSR with its rows ascending, and
// `D.T @ A` is `(A.T @ D).T`.  The multiply and the add are __fmul_rn / __fadd_rn so that nothing is contracted to
// an FFMA, which would round once instead of twice.
//
// A work unit is one row and one slice of 32 columns (one column per lane), so a row of W columns is ceil(W / 32)
// units on as many warps.  A long row is therefore split by columns, never by nonzeros: a split by nonzeros would
// need partial sums and so a different rounding.  Each lane's sum is one sequential chain, so the only parallelism
// inside a unit is memory-level: the warp reads 32 nonzeros at a time (one per lane), broadcasts them by shuffles
// and issues all 32 gathers before the 32 adds.  The grid is persistent and walks the units in the order d_order
// gives (rows longest first), so the longest rows start first and the short ones fill in behind them.
#include <algorithm>

#include "common.cuh"

namespace lk {

constexpr int SPMM_CT = 256;  // threads per CTA
constexpr int SPMM_WARPS = SPMM_CT / 32;
// three CTAs per SM leave 80 registers, enough for the 32 gathers in flight without spills (at 64 it spills)
constexpr int SPMM_MIN_CTAS = 3;

__global__ void __launch_bounds__(SPMM_CT, SPMM_MIN_CTAS) spmm_kernel(const lk_spmm_args a)
{
    const int lane = threadIdx.x & 31;
    const int W = a.width;
    const int S = (W + 31) >> 5;  // column slices per row
    const int64_t units = (int64_t)a.n_rows * S;
    const int64_t stride = (int64_t)gridDim.x * SPMM_WARPS;
    for (int64_t w = (int64_t)blockIdx.x * SPMM_WARPS + (threadIdx.x >> 5); w < units; w += stride) {
        const int row = __ldg(a.d_order + w / S);
        const int col = (int)(w % S) * 32 + lane;
        const bool on = col < W;
        const int b = __ldg(a.d_indptr + row), e = __ldg(a.d_indptr + row + 1);
        const float *dcol = a.d_dense + col;
        float acc = 0.0f;
        for (int64_t p0 = b; p0 < e; p0 += 32) {  // 64-bit: p0 + 32 may pass 2^31 - 1
            const int cnt = e - p0 < 32 ? (int)(e - p0) : 32;
            int j = 0;
            float v = 0.0f;
            if (lane < cnt) {
                j = ld_stream_s32(a.d_indices + p0 + lane);
                v = ld_stream_f32(a.d_values + p0 + lane);
            }
            float x[32];
#pragma unroll
            for (int u = 0; u < 32; u++) {
                const int ju = __shfl_sync(FULL, j, u);
                x[u] = on && u < cnt ? __ldg(dcol + (int64_t)ju * W) : 0.0f;
            }
            // the slots past cnt add +0.0f * +0.0f, which leaves acc as it is: acc starts at +0.0f and a sum
            // rounded to nearest is -0.0f only when both addends are, so acc is never -0.0f
#pragma unroll
            for (int u = 0; u < 32; u++) acc = __fadd_rn(acc, __fmul_rn(__shfl_sync(FULL, v, u), x[u]));
        }
        if (on) a.d_out[(int64_t)row * W + col] = acc;
    }
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_spmm(const lk_spmm_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_spmm: null args");
    const lk_spmm_args &a = *args;
    LK_REQUIRE(a.n_rows >= 0 && a.n_src >= 0 && a.width >= 1, LK_ERR_INVALID,
               "lk_spmm: n_rows and n_src must be non-negative and width positive");
    LK_REQUIRE(a.nnz >= 0 && a.nnz < 0x80000000LL, LK_ERR_UNSUPPORTED,
               "lk_spmm: nnz must be below 2^31 (int32 offsets)");
    const int64_t S = (a.width + 31) / 32;
    LK_REQUIRE((int64_t)a.n_src * a.width < (1LL << 62) && (int64_t)a.n_rows * a.width < (1LL << 62),
               LK_ERR_UNSUPPORTED, "lk_spmm: dense operands too large");
    if (a.n_rows == 0) return LK_OK;
    LK_REQUIRE(a.d_indptr && a.d_order && a.d_out, LK_ERR_INVALID, "lk_spmm: null input or output");
    LK_REQUIRE(a.nnz == 0 || (a.d_indices && a.d_values && a.d_dense), LK_ERR_INVALID, "lk_spmm: null input");
    static int occ = -1;
    if (occ < 0) LK_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spmm_kernel, SPMM_CT, 0));
    const int64_t want = ((int64_t)a.n_rows * S + SPMM_WARPS - 1) / SPMM_WARPS;
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>((int64_t)sm_count() * std::max(occ, 1), want));
    spmm_kernel<<<(unsigned)grid, SPMM_CT, 0, static_cast<cudaStream_t>(stream)>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
