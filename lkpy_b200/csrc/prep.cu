// prep.cu — item-kNN input preparation on the device (SURVEY.md §8f N4).
//
// Replaces the host stage of ItemKNNScorer.train, src/lenskit/knn/item.py:202-228
// (_center_ratings, _normalize_rows: SciPy / NumPy), which on ML-25M-shaped data takes 45x
// longer than the similarity build it feeds.  The f32 values it produces are the *inputs* of a
// bit-exact kernel, so this kernel reproduces the host arithmetic to the bit:
//
//   sums[i]   = np.add.reduceat(data_f32)           NumPy's float32 pairwise summation
//   means[i]  = float32(float64(sums[i]) / count)   np.divide(f32, int64, out=f32)
//   c         = data - means[i]                     float32
//   norms[i]  = sqrt(np.add.reduceat(float64(c)**2))  float64 pairwise summation
//   out       = float32(float64(c) * (1.0 / max(norms[i], FLT_MIN)))
//
// The sums follow NumPy's pairwise order (pairwise.cuh), every add an explicit round-to-nearest intrinsic.
// tests/test_prep_gpu.py compares the result bit for bit with lkpy_b200.data.knn_item_matrices
// (the SciPy calls of the reference).
//
// One thread per item column: the columns are independent, a column's pairwise tree is walked
// depth-first (eight independent accumulators per leaf give the memory-level parallelism).

#include <algorithm>

#include "common.cuh"
#include "pairwise.cuh"

namespace lk {

__global__ void __launch_bounds__(128) knn_prep_columns_kernel(const int32_t *__restrict__ indptr,
                                                             const float *__restrict__ vals, int n_cols,
                                                             int centre, float *__restrict__ means,
                                                             float *__restrict__ out)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_cols; i += gridDim.x * blockDim.x) {
        const int64_t lo = indptr[i];
        const int64_t n = (int64_t)indptr[i + 1] - lo;
        float mean = 0.0f;
        if (centre && n > 0) {
            const float s = segment_reduce<F32Ops>([&](int64_t p) { return __ldg(vals + p); }, lo, n);
            mean = __double2float_rn(__ddiv_rn((double)s, (double)n));
        }
        if (means != nullptr) means[i] = mean;
        if (n == 0) continue;
        auto centred = [&](int64_t p) { return centre ? __fsub_rn(__ldg(vals + p), mean) : __ldg(vals + p); };
        const double s2 = segment_reduce<F64Ops>(
            [&](int64_t p) {
                const double c = (double)centred(p);
                return __dmul_rn(c, c);
            },
            lo, n);
        const double norm = sqrt(s2);  // IEEE: correctly rounded
        const double recip = __ddiv_rn(1.0, fmax(norm, (double)1.17549435e-38f));
        for (int64_t p = lo; p < lo + n; p++) out[p] = __double2float_rn(__dmul_rn((double)centred(p), recip));
    }
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_knn_prep_columns(const int32_t *d_indptr, const float *d_vals, int32_t n_cols, int32_t centre,
                        float *d_means, float *d_out, void *stream)
{
    LK_REQUIRE(d_indptr && d_vals && d_out && n_cols >= 0, LK_ERR_INVALID, "lk_knn_prep_columns: bad arguments");
    if (n_cols == 0) return LK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int blocks = std::min((n_cols + 127) / 128, sm_count() * 16);
    knn_prep_columns_kernel<<<blocks, 128, 0, st>>>(d_indptr, d_vals, n_cols, centre, d_means, d_out);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
