// pairwise.cuh — NumPy's float reduction order on the device, shared by prep.cu (per-column sums), basic.cu
// (the global mean of the bias model) and stochastic.cu (the softmax and linear normalisers).
//
// NumPy's reduction of a segment is first + pairwise(rest), where pairwise(a, n) adds sequentially for n < 8,
// keeps eight interleaved partial sums for n <= 128 (combined as ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)), then the
// tail sequentially), and otherwise splits at n/2 rounded down to a multiple of 8
// (numpy/_core/src/umath/loops_utils.h.src).  Every add is an explicit round-to-nearest intrinsic: no FMA
// contraction, no reassociation.
#pragma once

#include <stdint.h>

namespace lk {

struct F32Ops {
    using T = float;
    __device__ static T add(T a, T b) { return __fadd_rn(a, b); }
};
struct F64Ops {
    using T = double;
    __device__ static T add(T a, T b) { return __dadd_rn(a, b); }
};

// the split of an inner node of the pairwise tree (n > 128): the left child's length
__host__ __device__ __forceinline__ int64_t pairwise_split(const int64_t n)
{
    const int64_t n2 = n / 2;
    return n2 - n2 % 8;
}

// Descend the pairwise tree over n_total values along the d leading bits of path p (a set bit takes the right
// child), giving the node's range [lo, lo + n).  Returns false when the path runs into a leaf above depth d with path
// bits left that are not all zero: no such node exists.  Cutting the tree at depth d this way hands its 2^d subtrees
// to parallel walkers (basic.cu's mean, stochastic.cu's normaliser).
__host__ __device__ __forceinline__ bool pairwise_node(const int64_t n_total, const int d, const uint32_t p,
                                                       int64_t &lo, int64_t &n)
{
    lo = 0, n = n_total;
    for (int k = 0; k < d; k++) {
        if (n <= 128) return (p & ((1u << (d - k)) - 1u)) == 0u;
        const int64_t n2 = pairwise_split(n);
        if ((p >> (d - 1 - k)) & 1u)
            lo += n2, n -= n2;
        else
            n = n2;
    }
    return true;
}

// leaf of the pairwise tree (n <= 128)
template <typename Ops, typename Get>
__device__ __forceinline__ typename Ops::T pairwise_leaf(const Get &get, int64_t lo, int64_t n)
{
    using T = typename Ops::T;
    if (n < 8) {
        T res = (T)0;
        for (int64_t i = 0; i < n; i++) res = Ops::add(res, get(lo + i));
        return res;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = get(lo + j);
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] = Ops::add(r[j], get(lo + i + j));
    }
    T res = Ops::add(Ops::add(Ops::add(r[0], r[1]), Ops::add(r[2], r[3])),
                     Ops::add(Ops::add(r[4], r[5]), Ops::add(r[6], r[7])));
    for (; i < n; i++) res = Ops::add(res, get(lo + i));
    return res;
}

// pairwise(a[lo .. lo+n)) with element i produced by get(i): the recursion of NumPy's pairwise sum walked
// depth-first with an explicit stack — depth <= log2(n / 64) < 32
template <typename Ops, typename Get>
__device__ typename Ops::T pairwise_sum(const Get &get, int64_t lo, int64_t n)
{
    using T = typename Ops::T;
    struct Frame {
        int64_t lo, n;
        T left;
        int stage;  // 1: left child running, 2: right child running
    };
    Frame stk[32];
    int sp = 0;
    int64_t clo = lo, cn = n;
    for (;;) {
        // descend along left children to a leaf
        while (cn > 128) {
            stk[sp].lo = clo, stk[sp].n = cn, stk[sp].stage = 1;
            sp++;
            cn = pairwise_split(cn);
        }
        T res = pairwise_leaf<Ops>(get, clo, cn);
        // climb: a finished left child starts the right one, a finished right child closes the node
        for (;;) {
            if (sp == 0) return res;
            Frame &f = stk[sp - 1];
            if (f.stage == 1) {
                const int64_t n2 = pairwise_split(f.n);
                f.left = res;
                f.stage = 2;
                clo = f.lo + n2, cn = f.n - n2;
                break;
            }
            res = Ops::add(f.left, res);
            sp--;
        }
    }
}

// np.add.reduce / reduceat over one segment: first element, then += pairwise(rest)
template <typename Ops, typename Get>
__device__ typename Ops::T segment_reduce(const Get &get, int64_t lo, int64_t n)
{
    if (n == 1) return get(lo);
    return Ops::add(get(lo), pairwise_sum<Ops>(get, lo + 1, n - 1));
}

}  // namespace lk
