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

// System layouts of the one-warp solve (KP = 32, 64).  Row-major (FOLD = false): row stride KP + 4.  Folded
// (FOLD = true, the k = 64 bf16 uniform-confidence route, where the smaller buffer buys residency; the address
// arithmetic costs the other routes more than they would gain): only the lower 8 x 8 blocks are stored, the
// diagonal blocks in full (36 blocks at KP = 64, 10 at KP = 32).  Block row b (rows 8 b .. 8 b + 7) has b + 1 blocks and block row
// KP / 8 - 1 - b has KP / 8 - b, so the two share 8 physical rows of KP + 8 floats: the lower half of the block
// rows at the start of each physical row, the upper half after its partner's blocks.  The physical rows are
// CHOL_LD = KP + 12 floats apart, an odd number of 16-byte granules, so the eight rows that one quarter-warp's
// float4 access touches lie in distinct banks (as the row-major stride KP + 4 did).  The rows of one block row are
// consecutive physical rows, so (in both layouts) row 8 b + r is chol_off(8 b, jb) + r * CHOL_LD with a
// compile-time stride, and a row's blocks are contiguous: element (i, j) is at chol_off(i, 0) + j for every
// j < 8 (i / 8 + 1).  Returns the offset in floats of row i's 8-column block jb (jb <= i / 8 when folded).
template <int KP, bool FOLD>
constexpr int CHOL_LD = FOLD ? KP + 12 : KP + 4;

template <int KP, bool FOLD>
__host__ __device__ __forceinline__ constexpr int chol_off(int i, int jb)
{
    if constexpr (!FOLD) return i * CHOL_LD<KP, FOLD> + 8 * jb;
    constexpr int NB = KP / 8;
    const int b = i >> 3;
    const bool low = b < NB / 2;
    return ((low ? b : NB - 1 - b) * 8 + (i & 7)) * CHOL_LD<KP, FOLD> + 8 * (jb + (low ? 0 : NB - b));
}

// floats of the system buffer chol_solve<KP, NW, FOLD> factors
template <int KP, bool FOLD>
constexpr int SYS_FLOATS = FOLD ? KP / 2 * CHOL_LD<KP, FOLD> : KP * (KP + 4);

// A[i][j] (j <= i, or j in the diagonal 8 x 8 block) in the system buffer chol_solve<KP, NW, FOLD> factors
template <int KP, bool FOLD>
__device__ __forceinline__ float *sys_at(float *As, int i, int j)
{
    return As + chol_off<KP, FOLD>(i, 0) + j;
}

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

// a0 b0 + a1 b1 + a2 b2 + a3 b3 in one fixed expression shape: the sums of one 4-column panel
__device__ __forceinline__ float dot4(float a0, float b0, float a1, float b1, float a2, float b2, float a3, float b3)
{
    return a0 * b0 + a1 * b1 + a2 * b2 + a3 * b3;
}

// Trailing update of one of chol_solve_warp's last two tiles, cc = KP - 16 (W = 4) or KP - 8 (W = 2).  Only its
// N = KP - cc = 4 W rows i >= cc are below the diagonal, all in the last row group, so a whole-warp pass over
// them would leave 16 or 24 lanes idle.  Here 8 / W lanes share each row, each updating W of the tile's 8
// columns, and read the row's panel entries back from As (the panel step stored exactly the values it holds
// in registers).  Every element gets the same two dot4 subtractions, in the same order, as in the general
// tile loop, so the factor's bits do not change.  Rows above the tile are not touched: that part of the
// upper triangle is never read (and not stored when folded).
template <int KP, int W, bool FOLD>
__device__ __forceinline__ void chol_tile_shared(float *As, const int tid, const int j0, const int cc)
{
    constexpr int N = 4 * W;
    static_assert(W == 2 || W == 4, "16 rows x 4 columns or 8 rows x 2 columns per lane pair / quad");
    const int lane = tid & 31;
    const int i = cc + lane % N, c0 = (lane / N) * W;
    const float *xi = As + chol_off<KP, FOLD>(i, j0 >> 3);
    const float4 x0 = *reinterpret_cast<const float4 *>(xi);
    const float4 x1 = *reinterpret_cast<const float4 *>(xi + 4);
    float *ap = As + chol_off<KP, FOLD>(i, cc >> 3) + c0;
    float a[W];
    if constexpr (W == 4) {
        const float4 v = *reinterpret_cast<const float4 *>(ap);
        a[0] = v.x, a[1] = v.y, a[2] = v.z, a[3] = v.w;
    } else {
        const float2 v = *reinterpret_cast<const float2 *>(ap);
        a[0] = v.x, a[1] = v.y;
    }
#pragma unroll
    for (int c = 0; c < W; c++) {
        const float *lc = As + chol_off<KP, FOLD>(cc + c0 + c, j0 >> 3);
        const float4 l0 = *reinterpret_cast<const float4 *>(lc);
        const float4 l1 = *reinterpret_cast<const float4 *>(lc + 4);
        a[c] -= dot4(x0.x, l0.x, x0.y, l0.y, x0.z, l0.z, x0.w, l0.w);
        a[c] -= dot4(x1.x, l1.x, x1.y, l1.y, x1.z, l1.z, x1.w, l1.w);
    }
    if constexpr (W == 4)
        *reinterpret_cast<float4 *>(ap) = make_float4(a[0], a[1], a[2], a[3]);
    else
        *reinterpret_cast<float2 *>(ap) = make_float2(a[0], a[1]);
}

// One-warp systems (KP = 32, 64): the chol_solve contract below with 8-column panels.  Every lane
// factors the 8x8 diagonal block redundantly from broadcast reads, then solves the panel entries of its
// rows t and t + 32 into registers (x[q][0..7]), applies them to its right-hand side and updates the
// trailing matrix in tiles 8 columns wide, so each trailing element is read and written once per 8
// columns of the factor instead of once per 4.  The last two tiles, which have only 16 and 8 rows in the
// lower triangle, spread those rows' columns over the whole warp (chol_tile_shared).
//
// The arithmetic is that of 4-column panels, operation for operation: where the second half of a panel
// (columns 4..7) meets the first, the first half's contribution is one dot4 subtracted before the second
// half's own terms, exactly as a separate 4-column panel's trailing update would have left it.  The
// trailing update subtracts the two halves' dot4s in turn, and the back substitution handles each 8-unknown
// step as two 4-unknown ones.  So the factor, x and the status are bit-identical to a 4-column solve.  A
// pivot row runs the same recurrence as the rows below it, which reproduces the broadcast factor's row
// exactly (same operands in the same order); its entries right of the diagonal are stored as zero.  As holds
// the system in the layout FOLD selects (chol_off); the rows of one block row are LD floats apart.
template <int KP, bool FOLD>
__device__ __forceinline__ bool chol_solve_warp(float *As, float *ys, float *dinv, const int tid)
{
    constexpr int LD = CHOL_LD<KP, FOLD>, RPT = KP / 32, P = 8;
    static_assert(KP % P == 0 && RPT >= 1, "one warp, whole 8-column panels");
    bool bad = false;
    float yv[RPT];
#pragma unroll
    for (int q = 0; q < RPT; q++) yv[q] = ys[tid + q * 32];
    // where this lane's row i = tid + 32 q starts: folded, computed once; row-major, i * LD where it is used
    int ro[RPT];
#pragma unroll
    for (int q = 0; q < RPT; q++) ro[q] = FOLD ? chol_off<KP, FOLD>(tid + q * 32, 0) : 0;

    for (int j0 = 0; j0 < KP; j0 += P) {
        // pivot block: rows j0..j0+7 of columns j0..j0+7, a diagonal block of the system (only its lower
        // triangle is used)
        float l[P][P], inv[P], z[P];
        const float *pb = As + chol_off<KP, FOLD>(j0, j0 >> 3);  // the pivot block
#pragma unroll
        for (int r = 0; r < P; r++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (4 * h > r) continue;
                const float4 v = *reinterpret_cast<const float4 *>(pb + r * LD + 4 * h);
                l[r][4 * h] = v.x, l[r][4 * h + 1] = v.y, l[r][4 * h + 2] = v.z, l[r][4 * h + 3] = v.w;
            }
        {
            const float4 y0 = *reinterpret_cast<const float4 *>(ys + j0);
            const float4 y1 = *reinterpret_cast<const float4 *>(ys + j0 + 4);
            z[0] = y0.x, z[1] = y0.y, z[2] = y0.z, z[3] = y0.w, z[4] = y1.x, z[5] = y1.y, z[6] = y1.z, z[7] = y1.w;
        }
        // dot4 of the first half's entries of rows r and c (c >= 4)
        auto lo4 = [&](const float(&a)[P], const float(&b)[P]) { return dot4(a[0], b[0], a[1], b[1], a[2], b[2], a[3], b[3]); };
#pragma unroll
        for (int r = 0; r < P; r++) {
#pragma unroll
            for (int c = 0; c < r; c++) {
                float s = l[r][c];
                if (c >= 4) s -= lo4(l[r], l[c]);
#pragma unroll
                for (int m = c & 4; m < c; m++) s -= l[r][m] * l[c][m];
                l[r][c] = s * inv[c];
            }
            float d = l[r][r];
            if (r >= 4) d -= lo4(l[r], l[r]);
#pragma unroll
            for (int m = r & 4; m < r; m++) d -= l[r][m] * l[r][m];
            bad |= !(d > 0.0f);  // NaN included
            inv[r] = rsqrt_nr(d);
            l[r][r] = d * inv[r];
            // forward substitution for the pivot rows
            float s = z[r];
            if (r >= 4) s -= lo4(l[r], z);
#pragma unroll
            for (int m = r & 4; m < r; m++) s -= l[r][m] * z[m];
            z[r] = s * inv[r];
        }
        __syncwarp();  // all reads of the diagonal block / pivot rhs precede their overwrite

        float x[RPT][P];
#pragma unroll
        for (int q = 0; q < RPT; q++) {
            const int i = tid + q * 32;
#pragma unroll
            for (int c = 0; c < P; c++) x[q][c] = 0.0f;
            if (i < j0) continue;
            float *ai = As + (FOLD ? ro[q] : i * LD) + j0;
            const float4 a0 = *reinterpret_cast<const float4 *>(ai);
            const float4 a1 = *reinterpret_cast<const float4 *>(ai + 4);
            const float av[P] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
            for (int c = 0; c < P; c++) {
                float s = av[c];
                if (c >= 4) s -= lo4(x[q], l[c]);
#pragma unroll
                for (int m = c & 4; m < c; m++) s -= x[q][m] * l[c][m];
                x[q][c] = s * inv[c];
            }
            if (i < j0 + P) {
                const int r = i - j0;
                float zr = z[0], ir = inv[0];
#pragma unroll
                for (int c = 1; c < P; c++) {
                    if (c == r) zr = z[c], ir = inv[c];
                    if (c > r) x[q][c] = 0.0f;
                }
                yv[q] = zr;
                dinv[i] = ir;
            } else {
                yv[q] -= lo4(x[q], z);
                yv[q] -= dot4(x[q][4], z[4], x[q][5], z[5], x[q][6], z[6], x[q][7], z[7]);
                if (i < j0 + 2 * P) ys[i] = yv[q];  // pivot rows of the next panel
            }
            *reinterpret_cast<float4 *>(ai) = make_float4(x[q][0], x[q][1], x[q][2], x[q][3]);
            *reinterpret_cast<float4 *>(ai + 4) = make_float4(x[q][4], x[q][5], x[q][6], x[q][7]);
        }
        __syncwarp();
        // Trailing update A[i][cc..cc+7] -= L[i][j0..j0+7] . L[cc..cc+7][j0..j0+7]^T for every row i and every
        // 8-column tile right of the panel, one 4-column half of the panel after the other.  Rows above a tile
        // (i < cc) only touch the upper triangle, which is never read; folded, it is not stored either, so they
        // skip the tile (row-major, the update is applied without a per-lane branch).  The loop is not unrolled:
        // unrolled by two it compiled to three copies of the tile body (about 400 more instructions per k = 64
        // kernel), and the ALS epoch ran 4-5 % slower (H100 80GB HBM3 at 700 W, DESIGN.md section 8).
#pragma unroll 1
        for (int cc = j0 + P; cc < KP - 2 * P; cc += P) {
            float4 L[P][2];
            const float *lb = As + chol_off<KP, FOLD>(cc, j0 >> 3);
#pragma unroll
            for (int c = 0; c < P; c++) {
                L[c][0] = *reinterpret_cast<const float4 *>(lb + c * LD);
                L[c][1] = *reinterpret_cast<const float4 *>(lb + c * LD + 4);
            }
#pragma unroll
            for (int q = 0; q < RPT; q++) {
                if (q * 32 + 31 < cc) continue;  // this whole row group is above the tile (uniform)
                const int i = tid + q * 32;
                if (FOLD && i < cc) continue;
                const float *xq = x[q];
                auto upd = [&](float a, const float4(&lc)[2]) {
                    a -= dot4(xq[0], lc[0].x, xq[1], lc[0].y, xq[2], lc[0].z, xq[3], lc[0].w);
                    a -= dot4(xq[4], lc[1].x, xq[5], lc[1].y, xq[6], lc[1].z, xq[7], lc[1].w);
                    return a;
                };
                float *ai = As + (FOLD ? ro[q] : i * LD) + cc;
                float4 a0 = *reinterpret_cast<float4 *>(ai);
                float4 a1 = *reinterpret_cast<float4 *>(ai + 4);
                a0.x = upd(a0.x, L[0]), a0.y = upd(a0.y, L[1]), a0.z = upd(a0.z, L[2]), a0.w = upd(a0.w, L[3]);
                a1.x = upd(a1.x, L[4]), a1.y = upd(a1.y, L[5]), a1.z = upd(a1.z, L[6]), a1.w = upd(a1.w, L[7]);
                *reinterpret_cast<float4 *>(ai) = a0;
                *reinterpret_cast<float4 *>(ai + 4) = a1;
            }
        }
        if (j0 + P <= KP - 2 * P) chol_tile_shared<KP, 4, FOLD>(As, tid, j0, KP - 2 * P);
        if (j0 + P <= KP - P) chol_tile_shared<KP, 2, FOLD>(As, tid, j0, KP - P);
        __syncwarp();
    }

    // back substitution L^T x = z, eight unknowns at a time from the bottom (as two steps of four); yv holds z
#pragma unroll
    for (int q = 0; q < RPT; q++) {
        const int i = tid + q * 32;
        if (i >= KP - P) ys[i] = yv[q];
    }
    __syncwarp();
    for (int j0 = KP - P; j0 >= 0; j0 -= P) {
        float l[P][P], xs[P], di[P];
        const float *rb = As + chol_off<KP, FOLD>(j0, 0);  // rows j0..j0+7 from column 0
#pragma unroll
        for (int r = 1; r < P; r++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (4 * h >= r) continue;
                const float4 v = *reinterpret_cast<const float4 *>(rb + r * LD + j0 + 4 * h);
                l[r][4 * h] = v.x, l[r][4 * h + 1] = v.y, l[r][4 * h + 2] = v.z, l[r][4 * h + 3] = v.w;
            }
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const float4 y = *reinterpret_cast<const float4 *>(ys + j0 + 4 * h);
            const float4 d = *reinterpret_cast<const float4 *>(dinv + j0 + 4 * h);
            xs[4 * h] = y.x, xs[4 * h + 1] = y.y, xs[4 * h + 2] = y.z, xs[4 * h + 3] = y.w;
            di[4 * h] = d.x, di[4 * h + 1] = d.y, di[4 * h + 2] = d.z, di[4 * h + 3] = d.w;
        }
        // the lower four unknowns, then their contribution to the upper four, then those
#pragma unroll
        for (int h = 1; h >= 0; h--) {
#pragma unroll
            for (int r = 4 * h + 3; r >= 4 * h; r--) {
                float s = xs[r];
#pragma unroll
                for (int m = r + 1; m < 4 * h + 4; m++) s -= l[m][r] * xs[m];
                xs[r] = s * di[r];
            }
            if (h == 1) {
#pragma unroll
                for (int r = 0; r < 4; r++) xs[r] -= dot4(l[4][r], xs[4], l[5][r], xs[5], l[6][r], xs[6], l[7][r], xs[7]);
            }
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < RPT; q++) {
            const int i = tid + q * 32;
            if (i < j0) {
                const float *col = rb + i;  // column i of rows j0..j0+7
                yv[q] -= dot4(col[4 * LD], xs[4], col[5 * LD], xs[5], col[6 * LD], xs[6], col[7 * LD], xs[7]);
                yv[q] -= dot4(col[0], xs[0], col[LD], xs[1], col[2 * LD], xs[2], col[3 * LD], xs[3]);
                if (i >= j0 - P) ys[i] = yv[q];  // pivot rows of the next (upper) panel
            } else if (i < j0 + P) {
                const int r = i - j0;
                float v = xs[0];
#pragma unroll
                for (int c = 1; c < P; c++)
                    if (c == r) v = xs[c];
                yv[q] = v;
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int q = 0; q < RPT; q++) ys[tid + q * 32] = yv[q];
    __syncwarp();
    return bad;
}

// Solve A x = y for a KP x KP SPD matrix held in shared memory (sys_at: row-major
// with row stride KP+4, lower triangle used, or folded lower blocks for one warp
// with FOLD), rhs in ys, scratch dinv[KP].  Executed
// by NW warps together.  Thread t owns rows t + q*32*NW and keeps their
// right-hand-side entries in registers.  On return ys holds x; the result is
// true when a pivot was not positive (LAPACK info != 0).  Only the lower
// triangle and the diagonal 16x16 blocks are read.
//
// NW == 1 runs chol_solve_warp.  Several warps (KP = 128): right-looking
// factorisation with 4-column panels: every thread factors the 4x4 diagonal
// block redundantly from broadcast reads, solves the panel entries of its own
// rows, applies the panel to its right-hand side (the forward substitution is
// fused into the factorisation), then updates the trailing matrix in 4x4 tiles.
// The back substitution L^T x = z runs panel by panel from the bottom.
template <int KP, int NW, bool FOLD = false>
__device__ __forceinline__ bool chol_solve(float *As, float *ys, float *dinv, const int tid)
{
    static_assert(!FOLD || NW == 1, "only the one-warp solve has a folded layout");
    if constexpr (NW == 1) return chol_solve_warp<KP, FOLD>(As, ys, dinv, tid);
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

// The entries of `this` row that thread tid writes back, for write_row's x_old.  The k = 64 tensor-core kernel
// reads them before its Cholesky, so that the global load's latency overlaps the solve instead of following it;
// nothing else writes the row while the CTA solves it.
template <int KP, int NW>
__device__ __forceinline__ void read_old_row(const float *thisrow, const int k, const int tid, float (&xold)[KP / (NW * 32)])
{
    constexpr int NT = NW * 32;
#pragma unroll
    for (int q = 0; q < KP / NT; q++) xold[q] = tid + q * NT < k ? thisrow[tid + q * NT] : 0.0f;
}

// Write x (in ys) to the row of `this` (and its replicas on peer GPUs) and add
// |x - x_old|^2 to the delta accumulator; a failed solve leaves the row
// untouched and records the row in the status word.  x_old is read from the
// row here, or comes from read_old_row when the kernel read it earlier (xold).
template <int KP, int NW>
__device__ __forceinline__ void write_row(const lk_als_args &a, const int row, float *thisrow,
                                          const float *ys, const int tid, bool bad, const float *xold = nullptr)
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
            const float d = xn - (xold ? xold[q] : thisrow[i]);
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
