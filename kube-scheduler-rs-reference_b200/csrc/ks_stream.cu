// ks_stream.cu — K3: in-batch conflict resolution + capacity commit for streaming reconcile (config C5).
// Mirrors what the reference gets from re-LISTing bound pods per cell (/root/reference/src/predicates.rs:34-38):
// a later pod of the batch sees the capacity taken by earlier pods of the same batch.
#include "ks_internal.cuh"
#include "ks_launch.h"

#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace ks {

constexpr int STREAM_MAX = 4096; // claims per launch (one CTA sorts them in shared memory)

// The capacity commit of a batch of n claims, by one CTA of THREADS threads: (1) bitonic sort of (node, arrival) keys
// in key[] (room for n rounded up to a power of two); (2) one thread per node segment walks its claimants in arrival
// order: accept iff the request still fits, then decrement free[] (single writer per node: no atomics,
// deterministic).  node_of(i) is claim i's node or -1 for none, request(i, rc, rm) reads its request and
// accept(i, ok) records the verdict; a claim without a node is rejected without a walk.  free[] is read through L2
// (__ldcg): inside the cooperative kernel other CTAs read it and this CTA wrote it in earlier rounds.
template <uint32_t THREADS, class NodeOf, class Request, class Accept>
__device__ __forceinline__ void commit_claims(unsigned long long* key, uint32_t n, int64_t* free_cpu, int64_t* free_mem,
                                              NodeOf&& node_of, Request&& request, Accept&& accept) {
    uint32_t m = 1;
    while (m < n) m <<= 1;
    for (uint32_t i = threadIdx.x; i < m; i += THREADS) {
        unsigned long long k = ~0ull; // padding and "no claim" sort last
        if (i < n) {
            const int32_t nd = node_of(i);
            if (nd >= 0) k = ((unsigned long long)(uint32_t)nd << 32) | i;
            else accept(i, false);
        }
        key[i] = k;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= m; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < m / 2; i += THREADS) {
                const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const unsigned long long a = key[lo], b = key[hi];
                if ((a > b) == up) {
                    key[lo] = b;
                    key[hi] = a;
                }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < m; i += THREADS) {
        const unsigned long long k = key[i];
        if (k == ~0ull) continue;
        const uint32_t node = (uint32_t)(k >> 32);
        if (i > 0 && (uint32_t)(key[i - 1] >> 32) == node) continue; // not a segment head
        int64_t fc = __ldcg(free_cpu + node), fm = __ldcg(free_mem + node);
        for (uint32_t j = i; j < m && key[j] != ~0ull && (uint32_t)(key[j] >> 32) == node; j++) {
            const uint32_t c = (uint32_t)key[j];
            int64_t rc, rm;
            request(c, rc, rm);
            const bool ok = rc <= fc && rm <= fm; // predicates.rs:42 against what is left
            accept(c, ok);
            if (ok) { // util.rs:31-36
                fc -= rc;
                fm -= rm;
            }
        }
        free_cpu[node] = fc;
        free_mem[node] = fm;
    }
}

__global__ void __launch_bounds__(1024)
    k_stream_resolve(int64_t* __restrict__ free_cpu, int64_t* __restrict__ free_mem, const int32_t* __restrict__ claim_node,
                     const int64_t* __restrict__ req_cpu, const int64_t* __restrict__ req_mem, uint32_t n, uint32_t N,
                     uint8_t* __restrict__ accepted) {
    __shared__ unsigned long long key[STREAM_MAX];
    commit_claims<1024>(
        key, n, free_cpu, free_mem,
        [&](uint32_t i) {
            const int32_t nd = claim_node[i];
            return nd >= 0 && (uint32_t)nd < N ? nd : -1;
        },
        [&](uint32_t c, int64_t& rc, int64_t& rm) {
            rc = req_cpu[c];
            rm = req_mem[c];
        },
        [&](uint32_t c, bool ok) { accepted[c] = ok; });
}

cudaError_t launch_stream_resolve(int64_t* free_cpu, int64_t* free_mem, const int32_t* claim_node, const int64_t* req_cpu,
                                  const int64_t* req_mem, uint32_t n, uint32_t N, uint8_t* accepted, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    if (n > STREAM_MAX) return cudaErrorInvalidValue;
    k_stream_resolve<<<1, 1024, 0, st>>>(free_cpu, free_mem, claim_node, req_cpu, req_mem, n, N, accepted);
    g_launches++;
    return cudaGetLastError();
}

uint32_t stream_max_claims() { return STREAM_MAX; }

// ------------------------------------------------------------------------------------------------ device-side loop
// k_stream_batch: the whole micro-batch loop of ks_stream_bind in ONE cooperative launch (no host round trip per
// round).  Per round, exactly as the host loop / the oracle (orc_stream_bind_packed):
//   A  every CTA scans its slice of the node table for every pending pod (one warp per pod, lanes over nodes):
//      feasible (predicates.rs:42,45-61) -> policy key -> warp argmax (ties -> lowest node index) -> partial[pod][cta]
//   B  CTA 0 reduces the partials to one claim per pod, resolves the claims per node in arrival order against what
//      is left (commit_claims, as k_stream_resolve), writes the bindings and compacts the losers (order preserved)
//      into the next round's pending list
// separated by grid-wide barriers.  Batches of up to STREAM_BATCH_MAX pods.  The pods' requests, selectors and the
// node table are read-only here (__ldg); free[] changes between rounds and is read through L2 (__ldcg).
// Phases A and B are the two functions below; k_gang_batch runs the same rounds once per pod group.
constexpr uint32_t SB_THREADS = 256;

// Phase A of one round, every CTA: for the cnt pending pods of pl (indices into a's pod arrays), the best feasible
// node of this CTA's slice [n0, n1) into a.pkey / a.pidx [pod][cta]
template <int W>
__device__ __forceinline__ void stream_round_scan(const StreamBatchArgs& a, const uint32_t* pl, uint32_t cnt, uint32_t n0,
                                                  uint32_t n1, uint32_t G, uint32_t lane, uint32_t warp) {
    for (uint32_t k = warp; k < cnt; k += SB_THREADS / 32) {
        const uint32_t p = __ldcg(pl + k);
        const int64_t rc = __ldg(a.req_cpu + p), rm = __ldg(a.req_mem + p);
        uint64_t sw[W];
#pragma unroll
        for (int w = 0; w < W; w++) sw[w] = __ldg(a.sel + (size_t)p * W + w);
        int64_t best = INT64_MIN;
        int32_t bidx = -1;
        for (uint32_t n = n0 + lane; n < n1; n += 32) {
            const int64_t fc = __ldcg(a.free_cpu + n), fm = __ldcg(a.free_mem + n);
            uint64_t miss = 0;
#pragma unroll
            for (int w = 0; w < W; w++) miss |= sw[w] & ~__ldg(a.labels + (size_t)w * a.Npad + n);
            if (rc <= fc && rm <= fm && miss == 0) {
                const int64_t key = alloc_score_rt(a.policy, fc, fm, a.alloc_cpu, a.alloc_mem, n, rc, rm);
                if (key > best) { // ascending n per lane: strict '>' keeps the lowest index
                    best = key;
                    bidx = (int32_t)n;
                }
            }
        }
        warp_argmax(best, bidx);
        if (lane == 0) {
            a.pkey[(size_t)k * G + blockIdx.x] = best;
            a.pidx[(size_t)k * G + blockIdx.x] = bidx;
        }
    }
}

// Phase B of one round, CTA 0 only: reduce the partials to one claim per pod, commit the claims, write the winners'
// bindings into a.out_idx / a.out_score, compact the losers into the other pending list (a.pend half cur ^ 1) and
// publish (losers, round + 1) in a.ctl
template <int W>
__device__ __forceinline__ void stream_round_commit(const StreamBatchArgs& a, const uint32_t* pl, uint32_t cur,
                                                    uint32_t cnt, uint32_t round, uint32_t G, uint32_t tid,
                                                    uint32_t lane, uint32_t warp, unsigned long long* s_key,
                                                    int64_t* s_ckey, int32_t* s_claim, uint8_t* s_acc,
                                                    uint32_t* s_scan) {
    for (uint32_t k = warp; k < cnt; k += SB_THREADS / 32) {
        int64_t best = INT64_MIN;
        int32_t bidx = -1;
        for (uint32_t c = lane; c < G; c += 32) // ascending CTA = ascending node range
            merge_partial(best, bidx, __ldcg(a.pkey + (size_t)k * G + c), __ldcg(a.pidx + (size_t)k * G + c));
        warp_argmax(best, bidx);
        if (lane == 0) {
            s_claim[k] = bidx;
            s_ckey[k] = best;
        }
    }
    __syncthreads();
    // claims per node in arrival (batch) order
    commit_claims<SB_THREADS>(
        s_key, cnt, a.free_cpu, a.free_mem, [&](uint32_t k) { return s_claim[k]; },
        [&](uint32_t k, int64_t& rc, int64_t& rm) {
            const uint32_t p = __ldcg(pl + k);
            rc = __ldg(a.req_cpu + p);
            rm = __ldg(a.req_mem + p);
        },
        [&](uint32_t k, bool ok) { s_acc[k] = ok; });
    __syncthreads();
    // bindings of the winners; losers keep their order in the next pending list
    uint32_t* nl = a.pend + (cur ^ 1u) * STREAM_BATCH_MAX;
    constexpr uint32_t PER = STREAM_BATCH_MAX / SB_THREADS;
    uint32_t loser[PER], n_loser = 0;
#pragma unroll
    for (uint32_t e = 0; e < PER; e++) {
        const uint32_t k = tid * PER + e;
        loser[e] = 0;
        if (k < cnt && s_claim[k] >= 0) {
            const uint32_t p = __ldcg(pl + k);
            if (s_acc[k]) {
                a.out_idx[p] = s_claim[k];
                a.out_score[p] = key_score_rt(a.policy, s_ckey[k], a.req_cpu, a.req_mem, p);
            } else {
                loser[e] = 1;
                n_loser++;
            }
        }
    }
    s_scan[tid] = n_loser;
    __syncthreads();
    for (uint32_t off = 1; off < SB_THREADS; off <<= 1) { // inclusive scan (Hillis-Steele, 256 entries)
        const uint32_t v = tid >= off ? s_scan[tid - off] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    uint32_t pos = s_scan[tid] - n_loser;
#pragma unroll
    for (uint32_t e = 0; e < PER; e++)
        if (loser[e]) nl[pos++] = __ldcg(pl + tid * PER + e);
    if (tid == SB_THREADS - 1) {
        a.ctl[0] = s_scan[tid];
        a.ctl[1] = round + 1;
    }
    __threadfence();
}

template <int W>
__global__ void __launch_bounds__(SB_THREADS) k_stream_batch(const StreamBatchArgs a) {
    cg::grid_group grid = cg::this_grid();
    __shared__ unsigned long long s_key[STREAM_BATCH_MAX];
    __shared__ int64_t s_ckey[STREAM_BATCH_MAX];
    __shared__ int32_t s_claim[STREAM_BATCH_MAX];
    __shared__ uint8_t s_acc[STREAM_BATCH_MAX];
    __shared__ uint32_t s_scan[SB_THREADS];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x;
    const uint32_t chunk = (a.N + G - 1) / G, n0 = min(a.N, blockIdx.x * chunk), n1 = min(a.N, n0 + chunk);
    if (blockIdx.x == 0) {
        for (uint32_t i = tid; i < a.m; i += SB_THREADS) {
            a.pend[i] = i;
            a.out_idx[i] = -1; // NoNodeFound until bound (src/main.rs:116-118)
            a.out_score[i] = 0;
        }
        if (tid == 0) {
            a.ctl[0] = a.m;
            a.ctl[1] = 0;
        }
        __threadfence();
    }
    grid.sync();
    uint32_t cur = 0;
    for (uint32_t round = 0;; round++) {
        const uint32_t cnt = *reinterpret_cast<volatile uint32_t*>(a.ctl);
        if (cnt == 0 || round > a.max_rounds) break; // grid-uniform
        const uint32_t* pl = a.pend + cur * STREAM_BATCH_MAX;
        stream_round_scan<W>(a, pl, cnt, n0, n1, G, lane, warp);
        __threadfence();
        grid.sync();
        if (blockIdx.x == 0)
            stream_round_commit<W>(a, pl, cur, cnt, round, G, tid, lane, warp, s_key, s_ckey, s_claim, s_acc, s_scan);
        grid.sync();
        cur ^= 1u;
    }
}

// ------------------------------------------------------------------------------------------------ pod groups
// k_gang_batch: ks_gang_bind in ONE cooperative launch.  The groups run in order; group g is the pods
// [offset[g], offset[g+1]) of a's arrays, and its rounds are k_stream_batch's (phases A and B above) on a view of a
// shifted to the group, with the group's own control words ctl[2g..2g+1] (so no CTA can still be reading them when the
// next group starts).  After the last round CTA 0 counts the placed pods; if there are fewer than min_member[g] it
// rolls the group back: every placed pod's request is added back to free[] with 64-bit integer atomics (two's-complement
// sums do not depend on their order, so free[] returns bit for bit to its value before the group) and its binding
// becomes -1 / 0.  Then one grid barrier, and the next group sees the state the previous one left.
// a group's pods fill one pending list and the per-claim shared arrays, all STREAM_BATCH_MAX entries long
static_assert(KS_GANG_MAX_SIZE <= STREAM_BATCH_MAX, "a pod group must fit one cooperative micro-batch");

template <int W>
__global__ void __launch_bounds__(SB_THREADS, 1) k_gang_batch(const StreamBatchArgs a, const GangArgs ga) {
    cg::grid_group grid = cg::this_grid();
    __shared__ unsigned long long s_key[STREAM_BATCH_MAX];
    __shared__ int64_t s_ckey[STREAM_BATCH_MAX];
    __shared__ int32_t s_claim[STREAM_BATCH_MAX];
    __shared__ uint8_t s_acc[STREAM_BATCH_MAX];
    __shared__ uint32_t s_scan[SB_THREADS];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x;
    const uint32_t chunk = (a.N + G - 1) / G, n0 = min(a.N, blockIdx.x * chunk), n1 = min(a.N, n0 + chunk);
    for (uint32_t i = blockIdx.x * SB_THREADS + tid; i < a.m; i += G * SB_THREADS) {
        a.out_idx[i] = -1; // NoNodeFound until bound (src/main.rs:116-118)
        a.out_score[i] = 0;
    }
    for (uint32_t g = blockIdx.x * SB_THREADS + tid; g < ga.n; g += G * SB_THREADS) {
        ga.ctl[2 * g] = __ldg(ga.offset + g + 1) - __ldg(ga.offset + g);
        ga.ctl[2 * g + 1] = 0;
    }
    if (blockIdx.x == 0 && ga.n)
        for (uint32_t i = tid; i < __ldg(ga.offset + 1); i += SB_THREADS) a.pend[i] = i;
    __threadfence();
    grid.sync();
    for (uint32_t g = 0; g < ga.n; g++) {
        const uint32_t base = __ldg(ga.offset + g), size = __ldg(ga.offset + g + 1) - base;
        StreamBatchArgs b = a; // the group's view: its pods, its bindings, its control words
        b.req_cpu = a.req_cpu + base;
        b.req_mem = a.req_mem + base;
        b.sel = a.sel + (size_t)base * W;
        b.out_idx = a.out_idx + base;
        b.out_score = a.out_score + base;
        b.ctl = ga.ctl + 2 * g;
        b.m = size;
        b.max_rounds = size + 1;
        uint32_t cur = 0;
        for (uint32_t round = 0;; round++) {
            const uint32_t cnt = *reinterpret_cast<volatile uint32_t*>(b.ctl);
            if (cnt == 0 || round > b.max_rounds) break; // grid-uniform
            const uint32_t* pl = b.pend + cur * STREAM_BATCH_MAX;
            stream_round_scan<W>(b, pl, cnt, n0, n1, G, lane, warp);
            __threadfence();
            grid.sync();
            if (blockIdx.x == 0)
                stream_round_commit<W>(b, pl, cur, cnt, round, G, tid, lane, warp, s_key, s_ckey, s_claim, s_acc, s_scan);
            grid.sync();
            cur ^= 1u;
        }
        if (blockIdx.x == 0) {
            uint32_t placed = 0;
            for (uint32_t i0 = 0; i0 < size; i0 += SB_THREADS)
                placed += __syncthreads_count(i0 + tid < size && __ldcg(b.out_idx + i0 + tid) >= 0);
            if (placed < __ldg(ga.min_member + g)) { // roll back (placed is CTA-uniform)
                for (uint32_t i = tid; i < size; i += SB_THREADS) {
                    const int32_t nd = __ldcg(b.out_idx + i);
                    if (nd < 0) continue;
                    atomicAdd(reinterpret_cast<unsigned long long*>(a.free_cpu + nd), (unsigned long long)__ldg(b.req_cpu + i));
                    atomicAdd(reinterpret_cast<unsigned long long*>(a.free_mem + nd), (unsigned long long)__ldg(b.req_mem + i));
                    b.out_idx[i] = -1;
                    b.out_score[i] = 0;
                }
            }
            if (tid == 0) ga.placed[g] = placed;
            if (g + 1 < ga.n) // the next group starts from the pending list 0..size-1
                for (uint32_t i = tid; i < __ldg(ga.offset + g + 2) - __ldg(ga.offset + g + 1); i += SB_THREADS) a.pend[i] = i;
            __threadfence();
        }
        grid.sync();
    }
}

cudaError_t launch_gang_batch(const StreamBatchArgs& a, const GangArgs& g, uint32_t W, cudaStream_t st) {
    return with_label_width(W, [&](auto w) {
        StreamBatchArgs b = a;
        GangArgs h = g;
        void* args[] = {&b, &h};
        const cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(k_gang_batch<decltype(w)::value>),
                                                          dim3(a.grid), dim3(SB_THREADS), args, 0, st);
        if (e == cudaSuccess) g_launches++;
        return e;
    });
}

cudaError_t launch_stream_batch(const StreamBatchArgs& a, uint32_t W, cudaStream_t st) {
    return with_label_width(W, [&](auto w) {
        StreamBatchArgs b = a;
        void* args[] = {&b};
        const cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(k_stream_batch<decltype(w)::value>),
                                                          dim3(a.grid), dim3(SB_THREADS), args, 0, st);
        if (e == cudaSuccess) g_launches++;
        return e;
    });
}

} // namespace ks
