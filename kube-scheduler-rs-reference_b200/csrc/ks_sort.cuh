// ks_sort.cuh — block-wide scan and the stable in-CTA LSD radix pass shared by k_scaleup_pack (ks_scaleup.cu) and
// k_rep_order (ks_replicas.cu).  A CTA of 256 threads: one thread per 8-bit digit.
#pragma once
#include "ks_internal.cuh"

namespace ks {

constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;

struct SortShared {
    uint32_t hist[SORT_WARPS][256]; // per-warp digit counts, then per-warp digit cursors
    uint32_t wsum[SORT_WARPS];
};

// Exclusive block-wide prefix sum of v; all threads get the total.  Called by the whole CTA.
__device__ __forceinline__ uint32_t cta_block_scan(uint32_t v, uint32_t* wsum, uint32_t& total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, off);
        if (lane >= (uint32_t)off) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < SORT_WARPS; w++) {
        const uint32_t c = wsum[w];
        before += (uint32_t)w < warp ? c : 0u;
        all += c;
    }
    __syncthreads(); // wsum may be reused
    total = all;
    return before + x - v;
}

// One stable pass of the LSD radix sort, src[0, n) -> dst[0, n), on digit(element) in [0, 256).  Warp w owns a
// contiguous range of src, so the per-(digit, warp) cursors in that order give every element its stable position;
// inside a warp, equal digits are ranked by lane.  Called by the whole CTA.
template <class Digit>
__device__ __forceinline__ void cta_radix_pass(const uint32_t* src, uint32_t* dst, uint32_t n, Digit digit,
                                               SortShared& s) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t per = ((n + SORT_WARPS - 1) / SORT_WARPS + 31) & ~31u;
    const uint32_t lo = min(n, warp * per), hi = min(n, lo + per);
    for (uint32_t i = threadIdx.x; i < SORT_WARPS * 256; i += SORT_THREADS) (&s.hist[0][0])[i] = 0;
    __syncthreads();
    for (uint32_t i = lo + lane; i < hi; i += 32) atomicAdd(&s.hist[warp][digit(src[i])], 1u);
    __syncthreads();
    { // thread d: the cursors of digit d, warps in order
        const uint32_t d = threadIdx.x;
        uint32_t c[SORT_WARPS], sum = 0;
#pragma unroll
        for (int w = 0; w < SORT_WARPS; w++) {
            c[w] = s.hist[w][d];
            sum += c[w];
        }
        uint32_t total;
        uint32_t base = cta_block_scan(sum, s.wsum, total);
#pragma unroll
        for (int w = 0; w < SORT_WARPS; w++) {
            s.hist[w][d] = base;
            base += c[w];
        }
    }
    __syncthreads();
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t i0 = lo; i0 < hi; i0 += 32) { // warp-uniform bounds
        const uint32_t i = i0 + lane;
        const bool valid = i < hi;
        const uint32_t p = valid ? src[i] : 0u;
        const uint32_t d = valid ? digit(p) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & lt);
        const uint32_t pos = valid ? s.hist[warp][d] + rank : 0u;
        __syncwarp();
        if (valid && rank == 0) s.hist[warp][d] += __popc(peers);
        __syncwarp();
        if (valid) dst[pos] = p;
    }
    __syncthreads(); // dst is complete for the next pass
}

} // namespace ks
