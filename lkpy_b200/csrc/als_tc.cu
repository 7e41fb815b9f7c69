// als_tc.cu — ALS half-epoch with the Gram matrix on the tensor cores (sm_90a, mma.sync).
//
// Same contract as als_half_kernel (als_kernels.cu; reference src/accel/als/implicit.rs:87-125,
// explicit.rs:80-119) for k = 64 and k = 128, and the same shape of work: a persistent grid pulls
// chunks from the host plan, one CTA owns one chunk, the gathered rows are staged through shared
// memory by the TMA engine's bulk-copy path (cp.async.bulk + mbarrier), rows split over several chunks
// park partial systems in global memory and the last part sums them in slot order, and the k x k system
// is factored in shared memory (chol_solve, als_common.cuh).  What changes is the Gram:
//
//      z_j = s_j * other[c_j, :]      s_j = 1 (uniform weights / explicit) or sqrt(v_j)
//      G   = sum_j z_j z_j^T          on the tensor cores, fp32 accumulation in registers
//      implicit: A = OtOr + c * G     c = v (uniform) or 1;   y = sum_j (v_j + 1) o_j
//      explicit: A = G + reg * n * I                           y = sum_j v_j o_j
//
// Each warp owns a 64 x 64 quadrant of G as 4 x 8 m16n8 accumulator tiles (128 floats per lane, the
// SIMT kernel's register footprint); at k = 64 the one warp keeps only the 20 tiles the Cholesky reads (the
// lower triangle and the diagonal 16 x 16 blocks, 80 floats per lane), which lets 11-16 CTAs share an SM.
// A = Z^T and B = Z are the same staged tile:
//   * bf16 rows with unweighted / uniformly weighted Gram: mma.m16n8k16 bf16, operands loaded with
//     ldmatrix.trans (the tile is feature-contiguous, the MMA wants pairs along the gathered rows).
//     The products are exact; parity is against the oracle that rounds the gathered rows to bf16.
//   * fp32 rows, or per-nonzero confidences: every z is split exactly into hi = z with the low 13
//     mantissa bits cleared (a tf32 number) and lo = z - hi, and G is accumulated as
//     hi.hi + hi.lo + lo.hi with three mma.m16n8k8 tf32 per 8 gathered rows.  The dropped lo.lo term
//     and the tf32 truncation of lo are ~2^-22 relative per product, the size of the f32 rounding the
//     reference's own sgemm makes.
// Staged rows are KP + 8 elements apart, which makes both the ldmatrix row reads and the tf32 fragment
// reads bank-conflict free.  Rows past the end of a chunk read as zero (a zero row in shared memory for
// ldmatrix, a predicate for the scalar reads).

#include <algorithm>

#include "als_common.cuh"

namespace lk {

template <int KP, typename ET, int MODE, bool WEIGHTED>
struct TcCfg {
    using C = AlsCfg<KP>;
    static constexpr bool BF16MMA = sizeof(ET) == 2 && !WEIGHTED;
    // k = 64, bf16 rows, implicit feedback with a uniform confidence (the benchmark's route): every row's
    // right-hand-side weight is the same, so the kernel's rhs loop reads no values (RHS_PAIR in the kernel)
    static constexpr bool RHS_PAIR = BF16MMA && MODE == LK_ALS_IMPLICIT && KP == 64;
    static constexpr int SROW = KP + 8;  // staged row stride (elements)
    static constexpr int STAGE_ELTS = C::STAGE_ROWS * SROW;
    // the benchmark's route folds its system (chol_off) to fit 16 CTAs per SM
    static constexpr bool FOLD = RHS_PAIR;
    static constexpr int CHOL_BYTES = SYS_FLOATS<KP, FOLD> * 4;
    // Stages per route.  The benchmark's route keeps two, which with the folded system leaves room for 16 CTAs
    // per SM (OCC below).  The other k = 64 bf16 routes keep a third stage (two stages of look-ahead for the
    // gather) at 12 CTAs.
    static constexpr int NSTAGE = RHS_PAIR ? 2 : KP == 64 && sizeof(ET) == 2 ? 3 : C::NSTAGE;
    static constexpr int STAGES_BYTES = NSTAGE * STAGE_ELTS * (int)sizeof(ET);
    static constexpr int UNI = STAGES_BYTES > CHOL_BYTES ? STAGES_BYTES : CHOL_BYTES;
    static constexpr int ZERO_BYTES = KP * 2;  // one zero bf16 row (ldmatrix target for rows past the end)
    // union | y[KP] | dinv[KP] | zero row | mbarriers | misc
    static constexpr int ZERO_OFF = UNI + KP * 4 + KP * 4;
    static_assert(UNI % 16 == 0 && ZERO_OFF % 16 == 0, "bulk-copy destinations and ldmatrix rows are 16-byte aligned");
    static constexpr int SMEM_BYTES = ZERO_OFF + ZERO_BYTES + NSTAGE * 8 + 64;
    // k = 64: chol_solve reads only the lower triangle and the diagonal 16 x 16 blocks of the system, so the
    // one warp accumulates only the 20 m16n8 tiles (mi, nj) with nj <= 2 mi + 1 (80 floats per lane instead
    // of 128).  k = 128 keeps full 64 x 64 quadrants (a warp's quadrant may lie wholly in either triangle).
    static constexpr bool LOWER = KP == 64;
    __device__ static constexpr bool tile(int mi, int nj) { return !LOWER || nj <= 2 * mi + 1; }
    // CTAs per SM the registers allow.  Operand fragments sit next to the accumulators, so there are fewer
    // resident warps than in the SIMT kernel: at k = 64, 16 one-warp CTAs (128 registers each) on the
    // benchmark's route and 12 (168 registers) on the others, of which fp32 rows fit only 11 in shared memory;
    // 2 four-warp CTAs at k = 128 (up to 255 registers).
    static constexpr int OCC = KP >= 128 ? 2 : RHS_PAIR ? 16 : 12;
    // the folded route's 16 CTAs must also fit in shared memory: each takes the 1 KB the hardware reserves per
    // block besides SMEM_BYTES, of the SM's 228 KB
    static_assert(!FOLD || OCC * (SMEM_BYTES + 1024) <= 233472, "OCC CTAs fit one SM's shared memory");
};

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void mma_tf32_1688(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float tc_elt(float v) { return v; }
__device__ __forceinline__ float tc_elt(__nv_bfloat16 v) { return __bfloat162float(v); }

// exact split of z into a tf32 number and the f32 remainder
__device__ __forceinline__ void split_tf32(float z, uint32_t &hi, uint32_t &lo)
{
    hi = __float_as_uint(z) & 0xffffe000u;
    lo = __float_as_uint(z - __uint_as_float(hi));
}

// MODE: LK_ALS_IMPLICIT / LK_ALS_EXPLICIT.  ET: float or __nv_bfloat16 rows of `other`.  WEIGHTED: implicit
// mode with per-nonzero confidences (z = sqrt(v) o); otherwise the Gram is unweighted and scaled by the
// uniform confidence (implicit) or not at all (explicit).
template <int KP, typename ET, int MODE, bool WEIGHTED>
__global__ void __launch_bounds__(AlsCfg<KP>::NT, (TcCfg<KP, ET, MODE, WEIGHTED>::OCC)) als_tc_kernel(lk_als_args a)
{
    using C = AlsCfg<KP>;
    using T = TcCfg<KP, ET, MODE, WEIGHTED>;
    constexpr int NW = C::NW, NT = C::NT, SROW = T::SROW, NS = T::NSTAGE;
    constexpr bool IMPLICIT = MODE == LK_ALS_IMPLICIT;
    // k = 64, bf16 rows, uniform confidence v: every row's right-hand-side weight is the same v + 1, so the
    // loop over the rows needs no shuffle of the values, and lane l accumulates features 2 l and 2 l + 1 from
    // one 32-bit load per row
    constexpr bool RHS_PAIR = T::RHS_PAIR;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ET *stage0 = reinterpret_cast<ET *>(smem_raw);
    float *As = reinterpret_cast<float *>(smem_raw);
    float *ys = reinterpret_cast<float *>(smem_raw + T::UNI);
    float *dinv = ys + KP;
    unsigned char *zero_row = smem_raw + T::ZERO_OFF;
    uint64_t *bars = reinterpret_cast<uint64_t *>(zero_row + T::ZERO_BYTES);
    int *s_misc = reinterpret_cast<int *>(bars + NS);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    constexpr int k = KP;
    const ET *__restrict__ other = reinterpret_cast<const ET *>(a.d_other);
    constexpr uint32_t ROW_BYTES = (uint32_t)KP * sizeof(ET);
    // Gram quadrant of this warp
    const int qi = (warp / C::QUADS) * 64, qj = (warp % C::QUADS) * 64;
    const float scale = (IMPLICIT && !WEIGHTED) ? a.uniform_val : 1.0f;

    if (tid == 0) {
        for (int s = 0; s < NS; s++) mbar_init(&bars[s], 1);
        mbar_fence_init();
    }
    for (int i = tid; i < T::ZERO_BYTES / 16; i += NT) reinterpret_cast<uint4 *>(zero_row)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    uint32_t phases = 0;

    // k = 64: thread 0 claims the next chunk when it starts the current one, so the atomic's round trip
    // overlaps a whole chunk of work instead of leading the next one.  A claimed chunk is always finished:
    // after the cancel flag is raised, a CTA still completes the one chunk it has claimed ahead.
    constexpr bool CLAIM_AHEAD = KP == 64;
    int next = 0;
    if (CLAIM_AHEAD && tid == 0) next = fetch_work(a.d_work_counter, a.d_cancel);
    for (;;) {
        if (tid == 0) {
            if constexpr (CLAIM_AHEAD) {
                s_misc[0] = next;
                if (next < a.n_chunks) next = fetch_work(a.d_work_counter, a.d_cancel);
            } else {
                s_misc[0] = fetch_work(a.d_work_counter, a.d_cancel);
            }
        }
        __syncthreads();
        const int64_t ci = s_misc[0];
        __syncthreads();
        if (ci >= a.n_chunks) break;
        const int4 c0 = __ldg(reinterpret_cast<const int4 *>(a.d_chunks) + 2 * ci);
        const int row = c0.x, begin = c0.y, len = c0.z, nparts = c0.w;
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

        float acc[4][8][4];  // tiles outside T::tile are never touched
#pragma unroll
        for (int mi = 0; mi < 4; mi++)
#pragma unroll
            for (int nj = 0; nj < 8; nj++)
#pragma unroll
                for (int r = 0; r < 4; r++)
                    if (T::tile(mi, nj)) acc[mi][nj][r] = 0.0f;
        float yacc[C::YPT];
#pragma unroll
        for (int q = 0; q < C::YPT; q++) yacc[q] = 0.0f;
        float ypair[2] = {0.0f, 0.0f};  // RHS_PAIR: y[2 lane], y[2 lane + 1]
        const float wu = a.uniform_val + 1.0f;

        const int n_it = (len + 31) >> 5;
        const int32_t *cols = a.d_cols + begin;
        const float *vals = a.d_vals + begin;
        // column index of this lane's row in stages it .. it + NS (cq[0]: stage it), value in stages it, it + 1
        // (RHS_PAIR reads no values: they all equal the uniform confidence)
        int cq[NS + 1];
        float vq[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NS; j++) cq[j] = j * 32 + lane < len ? __ldg(cols + j * 32 + lane) : -1;
        if constexpr (!RHS_PAIR) {
#pragma unroll
            for (int j = 0; j < 2; j++) vq[j] = j * 32 + lane < len ? __ldg(vals + j * 32 + lane) : 0.f;
        }

        auto issue = [&](int it, int c) {
            const int s = it % NS;
            const int nrows = min(32, len - it * 32);
            ET *dst = stage0 + s * T::STAGE_ELTS;
            if (warp == 0) {
                if (lane == 0) mbar_arrive_expect_tx(&bars[s], (uint32_t)nrows * ROW_BYTES);
                if (lane < nrows) bulk_g2s(dst + lane * SROW, other + (size_t)c * k, ROW_BYTES, &bars[s]);
            }
        };

#pragma unroll
        for (int j = 0; j < NS - 1; j++)
            if (j < n_it) issue(j, cq[j]);
        for (int it = 0; it < n_it; it++) {
            const int s = it % NS;
            // column indices NS stages ahead
            const int nxt = (it + NS) * 32 + lane;
            cq[NS] = nxt < len ? __ldg(cols + nxt) : -1;
            const int vnxt = (it + 2) * 32 + lane;
            const float vn = !RHS_PAIR && vnxt < len ? __ldg(vals + vnxt) : 0.f;
            if (it + NS - 1 < n_it) issue(it + NS - 1, cq[NS - 1]);
            mbar_wait(&bars[s], (phases >> s) & 1u);
            phases ^= (1u << s);
            const int nrows = min(32, len - it * 32);
            const ET *st = stage0 + s * T::STAGE_ELTS;

            // right-hand side, as the SIMT kernel computes it: y = fma(o_r, w_r, y) over the rows in order
            if constexpr (RHS_PAIR) {
                for (int r = 0; r < nrows; r++) {
                    const uint32_t u = *reinterpret_cast<const uint32_t *>(st + r * SROW + 2 * lane);
                    ypair[0] = fmaf(__uint_as_float(u << 16), wu, ypair[0]);
                    ypair[1] = fmaf(__uint_as_float(u & 0xffff0000u), wu, ypair[1]);
                }
            } else {
                for (int r = 0; r < nrows; r++) {
                    const float v = __shfl_sync(FULL, vq[0], r);
                    const float w = IMPLICIT ? v + 1.0f : v;
#pragma unroll
                    for (int q = 0; q < C::YPT; q++) yacc[q] = fmaf(tc_elt(st[r * SROW + tid + q * NT]), w, yacc[q]);
                }
            }

            if constexpr (T::BF16MMA) {
                const uint32_t sbase = smem_u32(st), zaddr = smem_u32(zero_row);
                const int lr = lane & 7, lm = lane >> 3;
                for (int k0 = 0; k0 < nrows; k0 += 16) {
                    // A = Z^T: matrices (rows k0.., m0), (k0.., m0+8), (k0+8.., m0), (k0+8.., m0+8)
                    uint32_t af[4][4], bfr[4][4];
                    const int ra = k0 + lr + 8 * (lm >> 1);
#pragma unroll
                    for (int mi = 0; mi < 4; mi++) {
                        const int col = qi + 16 * mi + 8 * (lm & 1);
                        ldmatrix_x4_trans(af[mi], ra < nrows ? sbase + (uint32_t)((ra * SROW + col) * 2) : zaddr);
                    }
                    // B = Z: matrices (rows k0.., n0), (k0+8.., n0), (k0.., n0+8), (k0+8.., n0+8)
                    const int rb = k0 + lr + 8 * (lm & 1);
#pragma unroll
                    for (int np = 0; np < 4; np++) {
                        const int col = qj + 16 * np + 8 * (lm >> 1);
                        ldmatrix_x4_trans(bfr[np], rb < nrows ? sbase + (uint32_t)((rb * SROW + col) * 2) : zaddr);
                    }
#pragma unroll
                    for (int mi = 0; mi < 4; mi++)
#pragma unroll
                        for (int nj = 0; nj < 8; nj++)
                            if (T::tile(mi, nj))
                                mma_bf16_16816(acc[mi][nj], af[mi], bfr[nj >> 1][2 * (nj & 1)],
                                               bfr[nj >> 1][2 * (nj & 1) + 1]);
                }
            } else {
                const float sq = WEIGHTED ? sqrtf(vq[0]) : 1.0f;  // rows past the end carry v = 0
                for (int k0 = 0; k0 < nrows; k0 += 8) {
                    const int r0 = k0 + t, r1 = k0 + t + 4;
                    const bool ok0 = r0 < nrows, ok1 = r1 < nrows;
                    const float s0 = WEIGHTED ? __shfl_sync(FULL, sq, r0) : 1.0f;
                    const float s1 = WEIGHTED ? __shfl_sync(FULL, sq, r1) : 1.0f;
                    const ET *p0 = st + r0 * SROW, *p1 = st + r1 * SROW;
                    auto z = [&](bool ok, const ET *p, float s, int c) { return ok ? s * tc_elt(p[c]) : 0.0f; };
                    uint32_t bh[8][2], bl[8][2];
#pragma unroll
                    for (int nj = 0; nj < 8; nj++) {
                        split_tf32(z(ok0, p0, s0, qj + 8 * nj + g), bh[nj][0], bl[nj][0]);
                        split_tf32(z(ok1, p1, s1, qj + 8 * nj + g), bh[nj][1], bl[nj][1]);
                    }
#pragma unroll
                    for (int mi = 0; mi < 4; mi++) {
                        uint32_t ah[4], al[4];
                        const int m0 = qi + 16 * mi + g;
                        split_tf32(z(ok0, p0, s0, m0), ah[0], al[0]);
                        split_tf32(z(ok0, p0, s0, m0 + 8), ah[1], al[1]);
                        split_tf32(z(ok1, p1, s1, m0), ah[2], al[2]);
                        split_tf32(z(ok1, p1, s1, m0 + 8), ah[3], al[3]);
#pragma unroll
                        for (int nj = 0; nj < 8; nj++) {
                            if (!T::tile(mi, nj)) continue;
                            mma_tf32_1688(acc[mi][nj], ah, bh[nj][0], bh[nj][1]);
                            mma_tf32_1688(acc[mi][nj], ah, bl[nj][0], bl[nj][1]);
                            mma_tf32_1688(acc[mi][nj], al, bh[nj][0], bh[nj][1]);
                        }
                    }
                }
            }
            cta_sync<NW>();  // everyone is done with stage s before it is re-armed
#pragma unroll
            for (int j = 0; j < NS; j++) cq[j] = cq[j + 1];
            vq[0] = vq[1];
            vq[1] = vn;
        }

        if constexpr (RHS_PAIR) {
            // to the general layout: lane l holds y[l + 32 q], which lane (l >> 1) + 16 q holds in ypair[l & 1]
#pragma unroll
            for (int q = 0; q < C::YPT; q++) {
                const float y0 = __shfl_sync(FULL, ypair[0], (lane >> 1) + 16 * q);
                const float y1 = __shfl_sync(FULL, ypair[1], (lane >> 1) + 16 * q);
                yacc[q] = (lane & 1) ? y1 : y0;
            }
        }

        // accumulator (mi, nj, r) holds G[qi + 16 mi + g + 8 (r / 2)][qj + 8 nj + 2 t + r % 2]
        if (scale != 1.0f) {
#pragma unroll
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int nj = 0; nj < 8; nj++)
#pragma unroll
                    for (int r = 0; r < 4; r++)
                        if (T::tile(mi, nj)) acc[mi][nj][r] *= scale;
        }

        // ---- rows split over several chunks: park the partial, last part reduces
        if (nparts > 1) {
            // read here rather than with c0, so that it is not held through the Gram
            const int4 c1 = __ldg(reinterpret_cast<const int4 *>(a.d_chunks) + 2 * ci + 1);
            const int slot0 = c1.x, part = c1.y, split_idx = c1.z;
            float *slot = a.d_partials + (size_t)(slot0 + part) * C::SLOTF;
#pragma unroll
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int nj = 0; nj < 8; nj++)
#pragma unroll
                    for (int h = 0; h < 2; h++)
                        if (T::tile(mi, nj))
                            __stcg(reinterpret_cast<float2 *>(slot + (qi + 16 * mi + g + 8 * h) * KP + qj + 8 * nj + 2 * t),
                               make_float2(acc[mi][nj][2 * h], acc[mi][nj][2 * h + 1]));
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
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int nj = 0; nj < 8; nj++)
#pragma unroll
                    for (int r = 0; r < 4; r++)
                        if (T::tile(mi, nj)) acc[mi][nj][r] = 0.0f;
#pragma unroll
            for (int q = 0; q < C::YPT; q++) yacc[q] = 0.0f;
            for (int p = 0; p < nparts; p++) {
                const float *sp = a.d_partials + (size_t)(slot0 + p) * C::SLOTF;
#pragma unroll
                for (int mi = 0; mi < 4; mi++)
#pragma unroll
                    for (int nj = 0; nj < 8; nj++)
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            if (!T::tile(mi, nj)) continue;
                            const float2 v = __ldcg(
                                reinterpret_cast<const float2 *>(sp + (qi + 16 * mi + g + 8 * h) * KP + qj + 8 * nj + 2 * t));
                            acc[mi][nj][2 * h] += v.x;
                            acc[mi][nj][2 * h + 1] += v.y;
                        }
#pragma unroll
                for (int q = 0; q < C::YPT; q++) yacc[q] += __ldcg(sp + KP * KP + tid + q * NT);
            }
        }

        // ---- assemble A (+ OtOr | + reg*n*I) and y in shared memory
        const int n_row = __ldg(a.d_indptr + row + 1) - __ldg(a.d_indptr + row);
        const float regn = a.reg * (float)n_row;
#pragma unroll
        for (int mi = 0; mi < 4; mi++)
#pragma unroll
            for (int nj = 0; nj < 8; nj++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (!T::tile(mi, nj)) continue;
                    // folded: the upper 8 x 8 block of a diagonal 16 x 16 block is not stored (sys_at)
                    if (T::FOLD && nj == 2 * mi + 1 && h == 0) continue;
                    const int gi = qi + 16 * mi + g + 8 * h, gc = qj + 8 * nj + 2 * t;
                    float v0 = acc[mi][nj][2 * h], v1 = acc[mi][nj][2 * h + 1];
                    if constexpr (IMPLICIT) {
                        const float2 o = __ldg(reinterpret_cast<const float2 *>(a.d_otor + gi * k + gc));
                        v0 = o.x + v0;  // a = otor + mtm (implicit.rs:115)
                        v1 = o.y + v1;
                    } else {
                        if (gi == gc) v0 += regn;  // explicit.rs:106-108
                        if (gi == gc + 1) v1 += regn;
                    }
                    *reinterpret_cast<float2 *>(sys_at<KP, T::FOLD>(As, gi, gc)) = make_float2(v0, v1);
                }
#pragma unroll
        for (int q = 0; q < C::YPT; q++) ys[tid + q * NT] = yacc[q];
        cta_sync<NW>();

        // ---- Cholesky + triangular solves in shared memory, then write the row
        float xold[C::RPT];
        read_old_row<KP, NW>(thisrow, k, tid, xold);
        const bool bad = chol_solve<KP, NW, T::FOLD>(As, ys, dinv, tid);
        write_row<KP, NW>(a, row, thisrow, ys, tid, bad, xold);
        // the next chunk's bulk copies (async proxy) overwrite this buffer
        fence_proxy_async();
        __syncthreads();
    }
}

template <int KP, typename ET, int MODE, bool WEIGHTED>
static int launch_tc(const lk_als_args &a, cudaStream_t st)
{
    using T = TcCfg<KP, ET, MODE, WEIGHTED>;
    auto kern = als_tc_kernel<KP, ET, MODE, WEIGHTED>;
    LK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SMEM_BYTES));
    // k = 64 needs the whole 228 KB carve-out for 11-16 resident CTAs
    LK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int occ = 0;
    LK_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, AlsCfg<KP>::NT, T::SMEM_BYTES));
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>((int64_t)sm_count() * std::max(occ, 1), a.n_chunks));
    kern<<<(unsigned)grid, AlsCfg<KP>::NT, T::SMEM_BYTES, st>>>(a);
    LK_CUDA_TRY(cudaGetLastError());
    return LK_OK;
}

template <int KP, typename ET>
static int dispatch_tc(const lk_als_args &a, cudaStream_t st, bool weighted)
{
    if (a.mode == LK_ALS_EXPLICIT) return launch_tc<KP, ET, LK_ALS_EXPLICIT, false>(a, st);
    return weighted ? launch_tc<KP, ET, LK_ALS_IMPLICIT, true>(a, st) : launch_tc<KP, ET, LK_ALS_IMPLICIT, false>(a, st);
}

// returns LK_OK when the tensor-core kernel took the launch, 1 when the caller should use the SIMT kernel
int launch_als_tc(const lk_als_args &a, cudaStream_t st)
{
    if (a.k != 64 && a.k != 128) return 1;
    if (reinterpret_cast<uintptr_t>(a.d_other) % 16 != 0) return 1;
    const bool f32 = a.other_dtype == LK_DTYPE_F32;
    const bool weighted = a.mode == LK_ALS_IMPLICIT && !a.vals_uniform;
    // the weighted Gram uses z = sqrt(v) o: confidences must not be negative (the plan passes the minimum)
    if (weighted && !(a.uniform_val >= 0.0f)) return 1;
    // LK_ALS_TF32 = 0: fp32 rows and per-nonzero confidences stay on the SIMT kernel
    if ((f32 || weighted) && options().als_tf32 == 0) return 1;
    if (a.k == 64)
        return f32 ? dispatch_tc<64, float>(a, st, weighted) : dispatch_tc<64, __nv_bfloat16>(a, st, weighted);
    return f32 ? dispatch_tc<128, float>(a, st, weighted) : dispatch_tc<128, __nv_bfloat16>(a, st, weighted);
}

}  // namespace lk
