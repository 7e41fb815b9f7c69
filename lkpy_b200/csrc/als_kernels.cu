// als_kernels.cu — ALS half-epoch for sm_90a (SIMT kernel; the tensor-core kernel is als_tc.cu).
//
// Replaces the reference's per-row rayon task
//   src/accel/als/implicit.rs:87-125  (train_row_solve, implicit feedback)
//   src/accel/als/explicit.rs:80-119  (train_row_solve, explicit feedback)
//   src/accel/als/solve.rs:65-106     (LAPACK sposv)
// and the NumPy OtOr of src/lenskit/als/_implicit.py:177-184.
//
// Shape of the work: for every CSR row (n nonzeros, columns c_j, values v_j)
//   implicit:  A = OtOr + sum_j v_j o_j o_j^T     y = sum_j (v_j + 1) o_j
//   explicit:  A = sum_j o_j o_j^T + reg*n*I      y = sum_j v_j o_j
//   x = A^-1 y (Cholesky);  delta += |x - x_old|^2;  row <- x
// with o_j = other[c_j, :].  At k = 64 the Gram is 2*n*k^2 flop against n*k*4
// gathered bytes (31 flop/B): it sits above the fp32-SIMT ridge, so this
// kernel is FMA-issue bound, not HBM bound (DESIGN.md §kernels); the gather is
// staged through shared memory by the TMA engine's bulk-copy path
// (cp.async.bulk + mbarrier) so that no SM issue slots are spent on it.
//
// Decomposition (DESIGN.md): the host plan cuts rows into chunks of <= chunk_nnz
// nonzeros ordered longest-row-first; a persistent grid pulls chunks from an
// atomic counter.  One CTA owns one chunk: (KP/64)^2 warps each hold a 64x64
// quadrant of the Gram in registers (16x8 accumulators per lane; 32x32 in one
// warp at KP=32).  Rows split over several chunks park partial Grams in global
// memory; the last part to arrive sums them in slot order (bit-reproducible)
// and solves.  The k x k system is factored in shared memory by a right-looking
// Cholesky with 4-column panels.

#include <algorithm>
#include <numeric>
#include <vector>

#include "als_common.cuh"

namespace lk {

template <int KP, typename ET>
__host__ __device__ constexpr int als_smem_bytes()
{
    using C = AlsCfg<KP>;
    int stage = C::NSTAGE * C::STAGE_ROWS * KP * (int)sizeof(ET);
    int chol = KP * C::LDA * (int)sizeof(float);
    int uni = stage > chol ? stage : chol;
    // union | y[KP] | dinv[KP] | mbarriers | misc
    return uni + KP * 4 + KP * 4 + C::NSTAGE * 8 + 64;
}

__device__ __forceinline__ void load_row_frag(const float *m, float *dst, int n)
{
#pragma unroll
    for (int q = 0; q < n / 4; q++) {
        float4 t = *reinterpret_cast<const float4 *>(m + 4 * q);
        dst[4 * q + 0] = t.x;
        dst[4 * q + 1] = t.y;
        dst[4 * q + 2] = t.z;
        dst[4 * q + 3] = t.w;
    }
}

__device__ __forceinline__ void load_row_frag(const __nv_bfloat16 *m, float *dst, int n)
{
    if (n == 4) {
        uint2 t = *reinterpret_cast<const uint2 *>(m);
        dst[0] = __uint_as_float(t.x << 16);
        dst[1] = __uint_as_float(t.x & 0xffff0000u);
        dst[2] = __uint_as_float(t.y << 16);
        dst[3] = __uint_as_float(t.y & 0xffff0000u);
        return;
    }
#pragma unroll
    for (int q = 0; q < n / 8; q++) {
        uint4 t = *reinterpret_cast<const uint4 *>(m + 8 * q);
        dst[8 * q + 0] = __uint_as_float(t.x << 16);
        dst[8 * q + 1] = __uint_as_float(t.x & 0xffff0000u);
        dst[8 * q + 2] = __uint_as_float(t.y << 16);
        dst[8 * q + 3] = __uint_as_float(t.y & 0xffff0000u);
        dst[8 * q + 4] = __uint_as_float(t.z << 16);
        dst[8 * q + 5] = __uint_as_float(t.z & 0xffff0000u);
        dst[8 * q + 6] = __uint_as_float(t.w << 16);
        dst[8 * q + 7] = __uint_as_float(t.w & 0xffff0000u);
    }
}

__device__ __forceinline__ float elt_to_f32(float v) { return v; }
__device__ __forceinline__ float elt_to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

template <int KP, typename ET, int MODE, bool BULK>
__global__ void __launch_bounds__(AlsCfg<KP>::NT, AlsCfg<KP>::OCC) als_half_kernel(lk_als_args a)
{
    using C = AlsCfg<KP>;
    constexpr int NW = C::NW, NT = C::NT, TM = C::TM, TN = C::TN, LDA = C::LDA;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int STAGE_BYTES = C::STAGE_ROWS * KP * (int)sizeof(ET);
    constexpr int STAGES_TOTAL = C::NSTAGE * STAGE_BYTES;
    constexpr int CHOL_BYTES = KP * LDA * 4;
    constexpr int UNI = STAGES_TOTAL > CHOL_BYTES ? STAGES_TOTAL : CHOL_BYTES;
    ET *stage0 = reinterpret_cast<ET *>(smem_raw);
    float *As = reinterpret_cast<float *>(smem_raw);
    float *ys = reinterpret_cast<float *>(smem_raw + UNI);
    float *dinv = ys + KP;
    uint64_t *bars = reinterpret_cast<uint64_t *>(dinv + KP);
    int *s_misc = reinterpret_cast<int *>(bars + C::NSTAGE);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k = a.k;
    const ET *__restrict__ other = reinterpret_cast<const ET *>(a.d_other);
    const uint32_t row_bytes = (uint32_t)k * (uint32_t)sizeof(ET);

    // quadrant / lane tile origin inside the KP x KP Gram
    const int qi = (warp / C::QUADS) * C::QS, qj = (warp % C::QUADS) * C::QS;
    const int ti = qi + (lane >> 3) * TM;  // first Gram row of this lane
    const int tj = qj + (lane & 7) * TN;   // first Gram col of this lane

    if (tid == 0) {
        for (int s = 0; s < C::NSTAGE; s++) mbar_init(&bars[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    uint32_t phases = 0;

    for (;;) {
        if (tid == 0) s_misc[0] = fetch_work(a.d_work_counter, a.d_cancel);
        __syncthreads();
        const int64_t ci = s_misc[0];
        __syncthreads();
        if (ci >= a.n_chunks) break;
        const int4 c0 = __ldg(reinterpret_cast<const int4 *>(a.d_chunks) + 2 * ci);
        const int4 c1 = __ldg(reinterpret_cast<const int4 *>(a.d_chunks) + 2 * ci + 1);
        const int row = c0.x, begin = c0.y, len = c0.z, nparts = c0.w;
        const int slot0 = c1.x, part = c1.y, split_idx = c1.z;
        float *thisrow = a.d_this + (size_t)row * k;

        if (len == 0 && nparts == 1) {
            // empty row: x = 0, contributes nothing to the delta (implicit.rs:98-101)
            for (int i = tid; i < k; i += NT) {
                thisrow[i] = 0.0f;
                for (int r = 0; r < a.n_replicas; r++)
                    a.d_replicas[r][(size_t)(a.replica_row0 + row) * k + i] = 0.0f;
            }
            continue;
        }

        // pad columns k..KP-1 of the stage rows must read as zero; the Cholesky
        // buffer aliases the stages, so re-zero them for every chunk.
        if (k < KP) {
            for (int idx = tid; idx < C::NSTAGE * C::STAGE_ROWS * (KP - k); idx += NT) {
                int r = idx / (KP - k), c = k + idx % (KP - k);
                stage0[r * KP + c] = ET(0.0f);
            }
        }
        fence_proxy_async();
        cta_sync<NW>();

        // accumulators as column pairs (each component is one fma.rn, the same rounding as the
        // reference's per-element update)
        float2 acc2[TM][TN / 2];
#pragma unroll
        for (int i = 0; i < TM; i++)
#pragma unroll
            for (int c = 0; c < TN / 2; c++) acc2[i][c] = make_float2(0.0f, 0.0f);
        float yacc[C::YPT];
#pragma unroll
        for (int q = 0; q < C::YPT; q++) yacc[q] = 0.0f;

        const int n_it = (len + 31) >> 5;
        const int32_t *cols = a.d_cols + begin;
        const float *vals = a.d_vals + begin;
        int cA = -1, cB = -1, cC = -1;
        float vA = 0.f, vB = 0.f, vC = 0.f;
        if (lane < len) {
            cA = __ldg(cols + lane);
            vA = __ldg(vals + lane);
        }
        if (32 + lane < len) {
            cB = __ldg(cols + 32 + lane);
            vB = __ldg(vals + 32 + lane);
        }

        auto issue = [&](int it, int c) {
            const int s = it & 1;
            const int nrows = min(32, len - it * 32);
            ET *dst = stage0 + s * (C::STAGE_ROWS * KP);
            if constexpr (BULK) {
                if (warp == 0) {
                    if (lane == 0) mbar_arrive_expect_tx(&bars[s], (uint32_t)nrows * row_bytes);
                    if (lane < nrows)
                        bulk_g2s(dst + lane * KP, other + (size_t)c * k, row_bytes, &bars[s]);
                }
            } else {
                // k*sizeof(ET) not a multiple of 16: plain loads, element by element
                for (int r = warp; r < nrows; r += NW) {
                    int cr = __shfl_sync(FULL, c, r);
                    const ET *src = other + (size_t)cr * k;
                    for (int e = lane; e < k; e += 32) dst[r * KP + e] = src[e];
                }
            }
        };

        // an empty part must not arm a stage it never waits on (the phase bits would fall out of step)
        if (n_it > 0) issue(0, cA);
        for (int it = 0; it < n_it; it++) {
            const int s = it & 1;
            // column indices two stages ahead
            if ((it + 2) * 32 + lane < len) {
                cC = __ldg(cols + (it + 2) * 32 + lane);
                vC = __ldg(vals + (it + 2) * 32 + lane);
            } else {
                cC = -1;
                vC = 0.f;
            }
            if (it + 1 < n_it) issue(it + 1, cB);
            if constexpr (BULK) {
                mbar_wait(&bars[s], (phases >> s) & 1u);
                phases ^= (1u << s);
            } else {
                cta_sync<NW>();
            }
            const int nrows = min(32, len - it * 32);
            const ET *st = stage0 + s * (C::STAGE_ROWS * KP);
#pragma unroll 2
            for (int r = 0; r < nrows; r++) {
                const ET *m = st + r * KP;
                float ra[TM], cb[TN];
                load_row_frag(m + ti, ra, TM);
                load_row_frag(m + tj, cb, TN);
                const float v = __shfl_sync(FULL, vA, r);
                float w;
                if constexpr (MODE == LK_ALS_IMPLICIT) {
                    w = v + 1.0f;
#pragma unroll
                    for (int c = 0; c < TN; c++) cb[c] *= v;
                } else {
                    w = v;
                }
#pragma unroll
                for (int i = 0; i < TM; i++) {
#pragma unroll
                    for (int c = 0; c < TN / 2; c++) {
                        acc2[i][c].x = fmaf(ra[i], cb[2 * c], acc2[i][c].x);
                        acc2[i][c].y = fmaf(ra[i], cb[2 * c + 1], acc2[i][c].y);
                    }
                }
#pragma unroll
                for (int q = 0; q < C::YPT; q++)
                    yacc[q] = fmaf(elt_to_f32(m[tid + q * NT]), w, yacc[q]);
            }
            cta_sync<NW>();  // everyone is done with stage s before it is re-armed
            cA = cB;
            vA = vB;
            cB = cC;
            vB = vC;
        }

        float acc[TM][TN];
#pragma unroll
        for (int i = 0; i < TM; i++)
#pragma unroll
            for (int c = 0; c < TN / 2; c++) {
                acc[i][2 * c] = acc2[i][c].x;
                acc[i][2 * c + 1] = acc2[i][c].y;
            }

        // ---- rows split over several chunks: park the partial, last part reduces
        if (nparts > 1) {
            float *slot = a.d_partials + (size_t)(slot0 + part) * C::SLOTF;
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int c = 0; c < TN; c += 4) {
                    if constexpr (TN >= 4) {
                        float4 t = make_float4(acc[i][c], acc[i][c + 1], acc[i][c + 2], acc[i][c + 3]);
                        __stcg(reinterpret_cast<float4 *>(slot + (ti + i) * KP + tj + c), t);
                    }
                }
#pragma unroll
            for (int q = 0; q < C::YPT; q++) __stcg(slot + KP * KP + tid + q * NT, yacc[q]);
            __threadfence();
            __syncthreads();
            if (tid == 0) {
                int old = atomicAdd(a.d_split_counters + split_idx, 1);
                s_misc[1] = (old == nparts - 1);
            }
            __syncthreads();
            const bool last = s_misc[1] != 0;
            __syncthreads();
            if (!last) continue;
            __threadfence();
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int c = 0; c < TN; c++) acc[i][c] = 0.0f;
#pragma unroll
            for (int q = 0; q < C::YPT; q++) yacc[q] = 0.0f;
            for (int p = 0; p < nparts; p++) {
                const float *sp = a.d_partials + (size_t)(slot0 + p) * C::SLOTF;
#pragma unroll
                for (int i = 0; i < TM; i++)
#pragma unroll
                    for (int c = 0; c < TN; c += 4) {
                        float4 t = __ldcg(reinterpret_cast<const float4 *>(sp + (ti + i) * KP + tj + c));
                        acc[i][c] += t.x;
                        acc[i][c + 1] += t.y;
                        acc[i][c + 2] += t.z;
                        acc[i][c + 3] += t.w;
                    }
#pragma unroll
                for (int q = 0; q < C::YPT; q++) yacc[q] += __ldcg(sp + KP * KP + tid + q * NT);
            }
        }

        // ---- assemble A (+ OtOr | + reg*n*I) and y in shared memory
        const int n_row = __ldg(a.d_indptr + row + 1) - __ldg(a.d_indptr + row);
        const float regn = a.reg * (float)n_row;
#pragma unroll
        for (int i = 0; i < TM; i++) {
            const int gi = ti + i;
            float out[TN];
#pragma unroll
            for (int c = 0; c < TN; c++) {
                const int gc = tj + c;
                float v = acc[i][c];
                if (gi < k && gc < k) {
                    if constexpr (MODE == LK_ALS_IMPLICIT)
                        v = __ldg(a.d_otor + gi * k + gc) + v;  // a = otor + mtm (implicit.rs:115)
                    else if (gi == gc)
                        v += regn;  // explicit.rs:106-108
                } else {
                    v = (gi == gc) ? 1.0f : 0.0f;
                }
                out[c] = v;
            }
#pragma unroll
            for (int c = 0; c < TN; c += 4)
                *reinterpret_cast<float4 *>(As + gi * LDA + tj + c) =
                    make_float4(out[c], out[c + 1], out[c + 2], out[c + 3]);
        }
#pragma unroll
        for (int q = 0; q < C::YPT; q++) ys[tid + q * NT] = yacc[q];
        cta_sync<NW>();

        // ---- Cholesky + triangular solves in shared memory, then write the row
        const bool bad = chol_solve<KP, NW>(As, ys, dinv, tid);
        write_row<KP, NW>(a, row, thisrow, ys, tid, bad);
        // the next chunk's bulk copies (async proxy) overwrite this buffer
        fence_proxy_async();
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------
// OtOr = O^T O + reg I  (and the bf16 copy of O for the bf16-gather mode)
// ---------------------------------------------------------------------------

constexpr int OTOR_GRID = 296;
constexpr int OTOR_ROWS = 32;

template <int KP>
__global__ void __launch_bounds__(256) otor_partial_kernel(const float *__restrict__ other,
                                                          int64_t n, int k,
                                                          float *__restrict__ partial,
                                                          __nv_bfloat16 *__restrict__ obf)
{
    constexpr int TS = KP / 16;
    __shared__ float sm[OTOR_ROWS][KP + 1];
    const int tid = threadIdx.x;
    const int ti = (tid >> 4) * TS, tj = (tid & 15) * TS;
    float acc[TS][TS];
#pragma unroll
    for (int i = 0; i < TS; i++)
#pragma unroll
        for (int j = 0; j < TS; j++) acc[i][j] = 0.0f;
    const int64_t per = (n + gridDim.x - 1) / gridDim.x;
    const int64_t r0 = per * blockIdx.x, r1 = min(n, r0 + per);
    for (int64_t rb = r0; rb < r1; rb += OTOR_ROWS) {
        const int nr = (int)min((int64_t)OTOR_ROWS, r1 - rb);
        for (int idx = tid; idx < OTOR_ROWS * KP; idx += 256) {
            const int r = idx / KP, c = idx % KP;
            float v = 0.0f;
            if (r < nr && c < k) {
                v = other[(rb + r) * k + c];
                if (obf != nullptr) {
                    __nv_bfloat16 b = __float2bfloat16_rn(v);
                    obf[(rb + r) * k + c] = b;
                    v = __bfloat162float(b);
                }
            }
            sm[r][c] = v;
        }
        __syncthreads();
        for (int r = 0; r < nr; r++) {
            float ra[TS], cb[TS];
#pragma unroll
            for (int i = 0; i < TS; i++) ra[i] = sm[r][ti + i];
#pragma unroll
            for (int j = 0; j < TS; j++) cb[j] = sm[r][tj + j];
#pragma unroll
            for (int i = 0; i < TS; i++)
#pragma unroll
                for (int j = 0; j < TS; j++) acc[i][j] = fmaf(ra[i], cb[j], acc[i][j]);
        }
        __syncthreads();
    }
    float *out = partial + (size_t)blockIdx.x * KP * KP;
#pragma unroll
    for (int i = 0; i < TS; i++)
#pragma unroll
        for (int j = 0; j < TS; j++) out[(ti + i) * KP + tj + j] = acc[i][j];
}

__global__ void otor_reduce_kernel(const float *__restrict__ partial, int nblocks, int KP, int k,
                                   float reg, float *__restrict__ out)
{
    // a block of 8 warps owns 32 consecutive output elements: warp g sums the partials g, g+8, ...
    // (coalesced 128-byte reads), warp 0 adds the eight sums in fixed order — deterministic, and
    // an eighth of the dependent loads per thread of the one-thread-per-element version
    __shared__ float part[8][32];
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int e = blockIdx.x * 32 + lane;
    const bool live = e < k * k;
    const int i = live ? e / k : 0, j = live ? e % k : 0;
    float s = 0.0f;
    if (live)
        for (int b = g; b < nblocks; b += 8) s += partial[(size_t)b * KP * KP + i * KP + j];
    part[g][lane] = s;
    __syncthreads();
    if (g == 0 && live) {
        float t = part[0][lane];
#pragma unroll
        for (int w = 1; w < 8; w++) t += part[w][lane];
        if (i == j) t += reg;
        out[e] = t;
    }
}

int launch_als_tc(const lk_als_args &a, cudaStream_t st);  // als_tc.cu (k = 64 / 128: bf16 MMA, or tf32 x3 for fp32 rows / non-uniform weights)

static int pad_features(int k) { return k <= 32 ? 32 : k <= 64 ? 64 : k <= 128 ? 128 : -1; }

template <int KP, typename ET, int MODE, bool BULK>
static int launch_als(const lk_als_args &a, cudaStream_t st)
{
    using C = AlsCfg<KP>;
    auto kern = als_half_kernel<KP, ET, MODE, BULK>;
    const int smem = als_smem_bytes<KP, ET>();
    LK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int occ = 0;
    LK_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, C::NT, smem));
    if (occ < 1) occ = 1;
    int64_t grid = (int64_t)sm_count() * occ;
    if (grid > a.n_chunks) grid = a.n_chunks;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, C::NT, smem, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

template <int KP, typename ET>
static int dispatch_mode(const lk_als_args &a, cudaStream_t st)
{
    const bool bulk = ((size_t)a.k * sizeof(ET)) % 16 == 0 &&
                      (reinterpret_cast<uintptr_t>(a.d_other) % 16 == 0);
    if (a.mode == LK_ALS_IMPLICIT)
        return bulk ? launch_als<KP, ET, LK_ALS_IMPLICIT, true>(a, st)
                    : launch_als<KP, ET, LK_ALS_IMPLICIT, false>(a, st);
    return bulk ? launch_als<KP, ET, LK_ALS_EXPLICIT, true>(a, st)
                : launch_als<KP, ET, LK_ALS_EXPLICIT, false>(a, st);
}

template <typename ET>
static int dispatch_k(const lk_als_args &a, cudaStream_t st)
{
    switch (pad_features(a.k)) {
        case 32: return dispatch_mode<32, ET>(a, st);
        case 64: return dispatch_mode<64, ET>(a, st);
        case 128: return dispatch_mode<128, ET>(a, st);
        default: set_error("embedding size %d not supported (max 128)", a.k); return LK_ERR_UNSUPPORTED;
    }
}

}  // namespace lk

using namespace lk;

extern "C" {

int lk_als_max_features(void) { return 128; }

int64_t lk_als_slot_floats(int32_t k)
{
    int kp = pad_features(k);
    return kp < 0 ? -1 : (int64_t)kp * kp + kp;
}

static int plan_impl(const int32_t *indptr, int64_t n_rows, int32_t chunk_nnz, int64_t *n_chunks,
                     int64_t *n_split, int64_t *n_slots, int32_t *out)
{
    // chunk_nnz a multiple of 32: then plen <= chunk_nnz, so (parts - 1) * plen < n and no part is empty
    // or longer than chunk_nnz (other lengths can round plen up far enough to leave the last part empty)
    LK_REQUIRE(indptr != nullptr && n_rows >= 0 && chunk_nnz >= 32 && chunk_nnz % 32 == 0, LK_ERR_INVALID,
               "lk_als_plan: bad arguments (chunk_nnz must be a positive multiple of 32)");
    std::vector<int32_t> order((size_t)n_rows);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) {
        return (indptr[x + 1] - indptr[x]) > (indptr[y + 1] - indptr[y]);
    });
    int64_t nc = 0, ns = 0, nslot = 0;
    for (int64_t t = 0; t < n_rows; t++) {
        const int32_t r = order[t];
        const int32_t n = indptr[r + 1] - indptr[r];
        if (n > chunk_nnz) {
            const int32_t parts = (n + chunk_nnz - 1) / chunk_nnz;
            // equal parts, multiples of 32 nonzeros
            int32_t plen = ((n + parts - 1) / parts + 31) & ~31;
            int32_t done = 0;
            for (int32_t p = 0; p < parts; p++) {
                const int32_t l = std::min(plen, n - done);
                if (out) {
                    int32_t *c = out + 8 * nc;
                    c[0] = r, c[1] = indptr[r] + done, c[2] = l, c[3] = parts;
                    c[4] = (int32_t)nslot, c[5] = p, c[6] = (int32_t)ns, c[7] = 0;
                }
                done += l;
                nc++;
            }
            nslot += parts;
            ns++;
        } else {
            if (out) {
                int32_t *c = out + 8 * nc;
                c[0] = r, c[1] = indptr[r], c[2] = n, c[3] = 1;
                c[4] = 0, c[5] = 0, c[6] = 0, c[7] = 0;
            }
            nc++;
        }
    }
    if (n_chunks) *n_chunks = nc;
    if (n_split) *n_split = ns;
    if (n_slots) *n_slots = nslot;
    return LK_OK;
}

int lk_als_plan_size(const int32_t *h_indptr, int64_t n_rows, int32_t chunk_nnz, int64_t *n_chunks,
                     int64_t *n_split_rows, int64_t *n_slots)
{
    return plan_impl(h_indptr, n_rows, chunk_nnz, n_chunks, n_split_rows, n_slots, nullptr);
}

int lk_als_plan_fill(const int32_t *h_indptr, int64_t n_rows, int32_t chunk_nnz, int32_t *h_chunks)
{
    LK_REQUIRE(h_chunks != nullptr, LK_ERR_INVALID, "lk_als_plan_fill: null output");
    return plan_impl(h_indptr, n_rows, chunk_nnz, nullptr, nullptr, nullptr, h_chunks);
}

int lk_als_half_epoch(const lk_als_args *args, void *stream)
{
    LK_REQUIRE(args != nullptr, LK_ERR_INVALID, "lk_als_half_epoch: null args");
    const lk_als_args &a = *args;
    LK_REQUIRE(a.mode == LK_ALS_IMPLICIT || a.mode == LK_ALS_EXPLICIT, LK_ERR_INVALID, "bad mode");
    LK_REQUIRE(a.k >= 1 && a.n_rows >= 0 && a.n_other >= 0, LK_ERR_INVALID, "bad shape");
    LK_REQUIRE(a.d_indptr && a.d_this && a.d_other && a.d_chunks && a.d_work_counter &&
                   a.d_sqdelta && a.d_status,
               LK_ERR_INVALID, "lk_als_half_epoch: null pointer");
    LK_REQUIRE(a.mode != LK_ALS_IMPLICIT || a.d_otor != nullptr, LK_ERR_INVALID,
               "implicit mode needs d_otor");
    LK_REQUIRE(a.n_replicas >= 0 && a.n_replicas <= LK_MAX_REPLICAS, LK_ERR_INVALID,
               "bad replica count");
    LK_REQUIRE(a.n_split_rows == 0 || (a.d_partials && a.d_split_counters), LK_ERR_INVALID,
               "split rows need partial workspace");
    LK_REQUIRE(a.other_dtype == LK_DTYPE_F32 || a.other_dtype == LK_DTYPE_BF16, LK_ERR_INVALID,
               "bad other_dtype");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (a.n_chunks == 0) return LK_OK;
    LK_CUDA_TRY(cudaMemsetAsync(a.d_work_counter, 0, sizeof(int32_t), st));
    if (a.n_split_rows > 0)
        LK_CUDA_TRY(cudaMemsetAsync(a.d_split_counters, 0, sizeof(int32_t) * a.n_split_rows, st));
    // k = 64 / 128: tensor-core kernel (als_tc.cu) unless switched off (option LK_ALS_TC = 0) or the
    // configuration is outside what it covers (returns 1: fall through to the SIMT kernel)
    if (options().als_tc != 0) {
        const int rc = launch_als_tc(a, st);
        if (rc <= 0) return rc;
    }
    if (a.other_dtype == LK_DTYPE_F32) return dispatch_k<float>(a, st);
    return dispatch_k<__nv_bfloat16>(a, st);
}

int64_t lk_als_otor_scratch_floats(int32_t k)
{
    int kp = pad_features(k);
    return kp < 0 ? -1 : (int64_t)OTOR_GRID * kp * kp;
}

int lk_als_otor(const float *d_other, int64_t n_other, int32_t k, float reg, float *d_otor,
                void *d_other_bf16, float *d_scratch, void *stream)
{
    LK_REQUIRE(d_other && d_otor && d_scratch && k >= 1 && n_other >= 0, LK_ERR_INVALID,
               "lk_als_otor: bad arguments");
    const int kp = pad_features(k);
    LK_REQUIRE(kp > 0, LK_ERR_UNSUPPORTED, "embedding size %d not supported (max 128)", k);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int grid = (int)std::min<int64_t>(OTOR_GRID, std::max<int64_t>(1, (n_other + OTOR_ROWS - 1) / OTOR_ROWS));
    __nv_bfloat16 *obf = static_cast<__nv_bfloat16 *>(d_other_bf16);
    switch (kp) {
        case 32: otor_partial_kernel<32><<<grid, 256, 0, st>>>(d_other, n_other, k, d_scratch, obf); break;
        case 64: otor_partial_kernel<64><<<grid, 256, 0, st>>>(d_other, n_other, k, d_scratch, obf); break;
        default: otor_partial_kernel<128><<<grid, 256, 0, st>>>(d_other, n_other, k, d_scratch, obf); break;
    }
    LK_CUDA_TRY(cudaGetLastError());
    otor_reduce_kernel<<<(k * k + 31) / 32, 256, 0, st>>>(d_scratch, grid, kp, k, reg, d_otor);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

}  // extern "C"
