// als_common.cuh — pieces shared by the SIMT and tensor-core ALS kernels:
// the in-shared-memory Cholesky solve (role of LAPACK sposv, solve.rs:65-106)
// and the row write-back with the |x - x_old|^2 reduction (implicit.rs:121-124).
#pragma once

#include "common.cuh"

namespace lk {

// launch shape of the ALS kernels (als_kernels.cu, als_tc.cu): one CTA per chunk, one warp per 64x64
// quadrant of the Gram
template <int KP>
struct AlsCfg {
    static constexpr int QUADS = KP >= 64 ? KP / 64 : 1;
    static constexpr int NW = QUADS * QUADS;  // warps per CTA
    static constexpr int NT = NW * 32;
    static constexpr int QS = KP >= 64 ? 64 : 32;  // quadrant edge
    static constexpr int TM = QS / 4;              // accumulator rows per lane
    static constexpr int TN = QS / 8;              // accumulator cols per lane
    static constexpr int STAGE_ROWS = 32;
    static constexpr int NSTAGE = 2;
    static constexpr int LDA = KP + 4;   // Cholesky row stride (floats), 16B-aligned rows
    static constexpr int RPT = KP / NT;  // Cholesky rows per thread
    static constexpr int YPT = KP / NT;  // rhs elements per thread
    static constexpr int SLOTF = KP * KP + KP;
    // CTAs per SM the register file allows (168 regs x 32 lanes x NW warps)
    static constexpr int OCC = KP >= 128 ? 3 : 12;
};

template <int NW>
__device__ __forceinline__ void cta_sync()
{
    if constexpr (NW == 1)
        __syncwarp();
    else
        __syncthreads();
}

// 1/sqrt(x) to f32 rounding: MUFU.RSQ seed + one Newton step (the IEEE sqrtf +
// divide pair costs ~4x the issue slots and sits on every panel's critical path)
__device__ __forceinline__ float rsqrt_nr(float x)
{
    const float r = rsqrtf(x);
    const float h = 0.5f * x;
    return r * fmaf(-h * r, r, 1.5f);
}

// Solve A x = y for a KP x KP SPD matrix held row-major in shared memory with
// row stride KP+4 (lower triangle used), rhs in ys, scratch dinv[KP].  Executed
// by NW warps together (NW == 1: one warp, only __syncwarp).  Thread t owns rows
// t + q*32*NW and keeps their right-hand-side entries in registers.  On return
// ys holds x; the result is true when a pivot was not positive (LAPACK info != 0).
//
// Right-looking factorisation with 4-column panels: every thread factors the 4x4
// diagonal block redundantly from broadcast reads, solves the panel entries of its
// own rows, applies the panel to its right-hand side (the forward substitution is
// fused into the factorisation), then updates the trailing matrix in 4x4 tiles.
// The back substitution L^T x = z runs panel by panel from the bottom.
template <int KP, int NW>
__device__ __forceinline__ bool chol_solve(float *As, float *ys, float *dinv, const int tid)
{
    constexpr int NT = NW * 32;
    constexpr int LDA = KP + 4;
    constexpr int RPT = KP / NT;
    static_assert(RPT >= 1, "at most KP threads may share one system");
    bool bad = false;
    float yv[RPT];
#pragma unroll
    for (int q = 0; q < RPT; q++) yv[q] = ys[tid + q * NT];

    for (int j0 = 0; j0 < KP; j0 += 4) {
        const float a00 = As[(j0 + 0) * LDA + j0];
        const float a10 = As[(j0 + 1) * LDA + j0], a11 = As[(j0 + 1) * LDA + j0 + 1];
        const float a20 = As[(j0 + 2) * LDA + j0], a21 = As[(j0 + 2) * LDA + j0 + 1],
                    a22 = As[(j0 + 2) * LDA + j0 + 2];
        const float a30 = As[(j0 + 3) * LDA + j0], a31 = As[(j0 + 3) * LDA + j0 + 1],
                    a32 = As[(j0 + 3) * LDA + j0 + 2], a33 = As[(j0 + 3) * LDA + j0 + 3];
        const float y0 = ys[j0], y1 = ys[j0 + 1], y2 = ys[j0 + 2], y3 = ys[j0 + 3];
        const float i0 = rsqrt_nr(a00), l00 = a00 * i0;
        const float l10 = a10 * i0, l20 = a20 * i0, l30 = a30 * i0;
        const float d1 = a11 - l10 * l10;
        const float i1 = rsqrt_nr(d1), l11 = d1 * i1;
        const float l21 = (a21 - l20 * l10) * i1, l31 = (a31 - l30 * l10) * i1;
        const float d2 = a22 - l20 * l20 - l21 * l21;
        const float i2 = rsqrt_nr(d2), l22 = d2 * i2;
        const float l32 = (a32 - l30 * l20 - l31 * l21) * i2;
        const float d3 = a33 - l30 * l30 - l31 * l31 - l32 * l32;
        const float i3 = rsqrt_nr(d3), l33 = d3 * i3;
        bad |= !(a00 > 0.0f && d1 > 0.0f && d2 > 0.0f && d3 > 0.0f);
        // forward substitution for the four pivot rows
        const float z0 = y0 * i0;
        const float z1 = (y1 - l10 * z0) * i1;
        const float z2 = (y2 - l20 * z0 - l21 * z1) * i2;
        const float z3 = (y3 - l30 * z0 - l31 * z1 - l32 * z2) * i3;
        cta_sync<NW>();  // all reads of the diagonal block / pivot rhs precede their overwrite

        float x[RPT][4];
#pragma unroll
        for (int q = 0; q < RPT; q++) {
            const int i = tid + q * NT;
            x[q][0] = x[q][1] = x[q][2] = x[q][3] = 0.0f;
            if (i >= j0 + 4) {
                float4 ar = *reinterpret_cast<const float4 *>(As + i * LDA + j0);
                const float x0 = ar.x * i0;
                const float x1 = (ar.y - x0 * l10) * i1;
                const float x2 = (ar.z - x0 * l20 - x1 * l21) * i2;
                const float x3 = (ar.w - x0 * l30 - x1 * l31 - x2 * l32) * i3;
                x[q][0] = x0, x[q][1] = x1, x[q][2] = x2, x[q][3] = x3;
                *reinterpret_cast<float4 *>(As + i * LDA + j0) = make_float4(x0, x1, x2, x3);
                yv[q] -= x0 * z0 + x1 * z1 + x2 * z2 + x3 * z3;
                if (i < j0 + 8) ys[i] = yv[q];  // pivot rows of the next panel
            } else if (i >= j0) {
                const int r = i - j0;
                float4 lr = r == 0   ? make_float4(l00, 0.f, 0.f, 0.f)
                            : r == 1 ? make_float4(l10, l11, 0.f, 0.f)
                            : r == 2 ? make_float4(l20, l21, l22, 0.f)
                                     : make_float4(l30, l31, l32, l33);
                *reinterpret_cast<float4 *>(As + i * LDA + j0) = lr;
                dinv[i] = r == 0 ? i0 : r == 1 ? i1 : r == 2 ? i2 : i3;
                yv[q] = r == 0 ? z0 : r == 1 ? z1 : r == 2 ? z2 : z3;
            }
        }
        cta_sync<NW>();
        // Trailing update A[i][cc..cc+3] -= L[i][j0..j0+3] . L[cc..cc+3][j0..j0+3]^T for every row i
        // and every 4-column tile right of the panel.  Rows above a tile (i < cc) only touch the
        // never-read upper triangle and pivot rows carry x = 0, so the update is applied without a
        // per-lane branch; tiles are independent, so two are kept in flight for latency.
#pragma unroll 2
        for (int cc = j0 + 4; cc < KP; cc += 4) {
            const float4 L0 = *reinterpret_cast<const float4 *>(As + (cc + 0) * LDA + j0);
            const float4 L1 = *reinterpret_cast<const float4 *>(As + (cc + 1) * LDA + j0);
            const float4 L2 = *reinterpret_cast<const float4 *>(As + (cc + 2) * LDA + j0);
            const float4 L3 = *reinterpret_cast<const float4 *>(As + (cc + 3) * LDA + j0);
#pragma unroll
            for (int q = 0; q < RPT; q++) {
                if (q * NT + NT - 1 < cc) continue;  // this whole row group is above the tile (uniform)
                const int i = tid + q * NT;
                float4 av = *reinterpret_cast<float4 *>(As + i * LDA + cc);
                av.x -= x[q][0] * L0.x + x[q][1] * L0.y + x[q][2] * L0.z + x[q][3] * L0.w;
                av.y -= x[q][0] * L1.x + x[q][1] * L1.y + x[q][2] * L1.z + x[q][3] * L1.w;
                av.z -= x[q][0] * L2.x + x[q][1] * L2.y + x[q][2] * L2.z + x[q][3] * L2.w;
                av.w -= x[q][0] * L3.x + x[q][1] * L3.y + x[q][2] * L3.z + x[q][3] * L3.w;
                *reinterpret_cast<float4 *>(As + i * LDA + cc) = av;
            }
        }
        cta_sync<NW>();
    }

    // back substitution L^T x = z, four unknowns at a time from the bottom; yv holds z
#pragma unroll
    for (int q = 0; q < RPT; q++) {
        const int i = tid + q * NT;
        if (i >= KP - 4) ys[i] = yv[q];
    }
    cta_sync<NW>();
    for (int j0 = KP - 4; j0 >= 0; j0 -= 4) {
        const float l10 = As[(j0 + 1) * LDA + j0];
        const float l20 = As[(j0 + 2) * LDA + j0], l21 = As[(j0 + 2) * LDA + j0 + 1];
        const float l30 = As[(j0 + 3) * LDA + j0], l31 = As[(j0 + 3) * LDA + j0 + 1],
                    l32 = As[(j0 + 3) * LDA + j0 + 2];
        const float x3 = ys[j0 + 3] * dinv[j0 + 3];
        const float x2 = (ys[j0 + 2] - l32 * x3) * dinv[j0 + 2];
        const float x1 = (ys[j0 + 1] - l21 * x2 - l31 * x3) * dinv[j0 + 1];
        const float x0 = (ys[j0] - l10 * x1 - l20 * x2 - l30 * x3) * dinv[j0];
        cta_sync<NW>();
#pragma unroll
        for (int q = 0; q < RPT; q++) {
            const int i = tid + q * NT;
            if (i < j0) {
                yv[q] -= As[(j0 + 0) * LDA + i] * x0 + As[(j0 + 1) * LDA + i] * x1 +
                         As[(j0 + 2) * LDA + i] * x2 + As[(j0 + 3) * LDA + i] * x3;
                if (i >= j0 - 4) ys[i] = yv[q];  // pivot rows of the next (upper) panel
            } else if (i < j0 + 4) {
                const int r = i - j0;
                yv[q] = r == 0 ? x0 : r == 1 ? x1 : r == 2 ? x2 : x3;
            }
        }
        cta_sync<NW>();
    }
#pragma unroll
    for (int q = 0; q < RPT; q++) ys[tid + q * NT] = yv[q];
    cta_sync<NW>();
    return bad;
}

// Write x (in ys) to the row of `this` (and its replicas on peer GPUs) and add
// |x - x_old|^2 to the delta accumulator; a failed solve leaves the row
// untouched and records the row in the status word.
template <int KP, int NW>
__device__ __forceinline__ void write_row(const lk_als_args &a, const int row, float *thisrow,
                                          const float *ys, const int tid, bool bad)
{
    constexpr int NT = NW * 32;
    constexpr int RPT = KP / NT;
    const int lane = tid & 31;
    const int k = a.k;
    if constexpr (NW == 1)
        bad = __any_sync(FULL, bad);
    else
        bad = __syncthreads_or(bad);
    if (bad) {
        if (tid == 0) atomicCAS(a.d_status, 0, row + 1);
        return;
    }
    float d2 = 0.0f;
#pragma unroll
    for (int q = 0; q < RPT; q++) {
        const int i = tid + q * NT;
        if (i < k) {
            const float xn = ys[i];
            const float d = xn - thisrow[i];
            d2 = fmaf(d, d, d2);
            thisrow[i] = xn;
            for (int r = 0; r < a.n_replicas; r++)
                a.d_replicas[r][(size_t)(a.replica_row0 + row) * k + i] = xn;
        }
    }
    d2 = warp_sum(d2);
    if (lane == 0 && d2 != 0.0f) atomicAdd(a.d_sqdelta, (double)d2);
}

}  // namespace lk
