// ks_replicas.cuh — what a pod spec's copies see of one node, shared by replica placement (ks_replicas.cu) and its
// topology-spread form (ks_spread.cu): c_n, s_n(j) and the CTA reduction of their scans.
#pragma once
#include "ks_internal.cuh"

namespace ks {

constexpr int REP_THREADS = 256;
constexpr int REP_WARPS = REP_THREADS / 32;

// One node as a spec sees it: free values, allocatable (LEAST_ALLOCATED, MOST_ALLOCATED) and k_n.
struct RepNode {
    int64_t fc, fm, ac, am;
    uint32_t k;
};

// c_n: 0 unless copy 0's cell is KS_CELL_OK, else the copies the node's free holds (UINT64_MAX when both requests are 0).
// fc >= rc >= 0 and fm >= rm >= 0 when it is not 0, so the divisions are exact integer floors.
template <int W>
__device__ __forceinline__ uint64_t rep_copies(const NodeTable& nt, uint32_t n, int64_t rc, int64_t rm,
                                               const uint64_t (&sel)[W], RepNode& v) {
    v.fc = nt.free_cpu[n];
    v.fm = nt.free_mem[n];
    uint64_t miss = 0;
#pragma unroll
    for (int w = 0; w < W; w++) miss |= sel[w] & ~nt.labels[(uint64_t)w * nt.Npad + n];
    if (rc > v.fc || rm > v.fm || miss) return 0;
    uint64_t c = ~0ull;
    if (rc > 0) c = (uint64_t)(v.fc / rc);
    if (rm > 0) c = min(c, (uint64_t)(v.fm / rm));
    return c;
}

template <int W, int POL>
__device__ __forceinline__ void rep_node(const NodeTable& nt, uint32_t n, int64_t rc, int64_t rm, const uint64_t (&sel)[W],
                                         uint32_t R, RepNode& v, uint64_t& c) {
    c = rep_copies<W>(nt, n, rc, rm, sel, v);
    v.k = (uint32_t)min(c, (uint64_t)R);
    if (POL != KS_SCORE_LEFTOVER && v.k) {
        v.ac = nt.alloc_cpu[n];
        v.am = nt.alloc_mem[n];
    } else {
        v.ac = v.am = 0;
    }
}

// s_n(j): ks_select's score with j copies bound (j < c_n)
template <int POL>
__device__ __forceinline__ int64_t rep_score(const RepNode& v, int64_t rc, int64_t rm, uint32_t j) {
    const int64_t c = v.fc - (int64_t)j * rc, m = v.fm - (int64_t)j * rm;
    return key_score<POL>(POL == KS_SCORE_LEFTOVER ? leftover_key(c, m) : alloc_score<POL>(c, m, v.ac, v.am, rc, rm), rc, rm);
}

template <class T, class Op>
__device__ __forceinline__ T rep_reduce(T x, Op op, T* sh /* [REP_WARPS] */) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x = op(x, __shfl_xor_sync(0xffffffffu, x, off));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    T r = sh[0];
#pragma unroll
    for (int w = 1; w < REP_WARPS; w++) r = op(r, sh[w]);
    __syncthreads(); // sh may be reused
    return r;
}

} // namespace ks
