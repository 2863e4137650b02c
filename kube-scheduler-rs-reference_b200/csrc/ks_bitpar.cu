// ks_bitpar.cu — bit-parallel fused feasibility pass for sm_90a (design notes in ks_bitpar.h, DESIGN.md).
//
//   per snapshot   k_node_bound, k_node_splitters/_bucket/_scatter/_rank  sample sort: global position of every node in
//                                   free_cpu / free_mem / leftover-priority / least-allocated-bound order
//                  k_build_tiles    one tile of 256 nodes of an index in the column-block format (8 tiles per block):
//                                   prefix tables + label-pair columns, 256-byte lines in tile order; three indexes:
//                                   node order (staged in shared memory by the mask kernel), priority order and bound
//                                   order (read through L1/L2 by the argmax kernels, with their bucket arrays)
//                  k_build_ranks    rank tables: tile-local rank of every possible threshold (read through L1/L2)
//   per call       k_pod_ranks      request -> global rank threshold (splitters in smem + short global search) and the mask
//                                   kernel's 16-byte pod record, in pod order
//                  k_mask_rows      persistent, 1 CTA per SM; table blob staged by TMA bulk copies (cp.async.bulk + mbarrier);
//                                   8 lanes = the 256 bytes of one pod: rank load -> 2 table granules per resource (+ label
//                                   columns) -> AND -> two 128-bit stores per lane, each instruction one whole 128-byte line
//                                   per pod; counts by shuffle + one RED per pod and column block
//                  k_first_fit_head/_tail  argmax KS_SCORE_LEFTOVER = first feasible node in priority order (early exit)
//                  k_least_alloc    argmax KS_SCORE_LEAST_ALLOCATED: bound-ordered scan, exact scores, early exit
//                  k_most_alloc     argmax KS_SCORE_MOST_ALLOCATED: the same scan over its own order (built lazily)
//                  k_least_balanced argmax KS_SCORE_LEAST_BALANCED: the same scan over another order (built lazily)
// Semantics per cell are exactly predicates.rs:42 / :45-61 (see include/ksched.h); only the evaluation
// order differs, and every output is compared bit-for-bit with the oracle in tests/.
#include "ks_bitpar.h"
#include "ks_sort.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace ks {

// ------------------------------------------------------------------------------------------------ step trace
// KS_TRACE=1 (environment, read when the index is created): every kernel of a select stamps %globaltimer into a small
// device buffer - first CTA at its start, every CTA at its end (atomic max) - so that the timeline of one step can be read
// back with ks_last_trace (nsys is not available on the target boxes and ncu serialises the streams).  Off: one
// constant-bank load per CTA.
__constant__ unsigned long long* c_trace = nullptr;
enum TraceSlot : int {
    TR_RANKS_START = 0, TR_RANKS_END, TR_ARGMAX1_START, TR_ARGMAX1_END, TR_ARGMAX2_START, TR_ARGMAX2_END,
    TR_MASK_START, TR_MASK_END, TR_MASK_FIRST_CTA_END_INV, TR_SLOTS
};
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// call with one thread per CTA
__device__ __forceinline__ void trace_start(int slot) {
    unsigned long long* tr = c_trace;
    if (tr && blockIdx.x == 0) tr[slot] = global_ns();
}
__device__ __forceinline__ void trace_end(int slot) {
    unsigned long long* tr = c_trace;
    if (tr) atomicMax(tr + slot, global_ns());
}

// ------------------------------------------------------------------------------------------------ build
// ---- node ranking: sample sort ------------------------------------------------------------------------------
// Three total orders over the N nodes are needed: ascending free_cpu, ascending free_mem, descending priority,
// ties always by node index.  All three are "ascending (v', index)" with v' = free_cpu, free_mem, -priority.
// k_node_splitters sorts 1024 sampled keys per order in shared memory and keeps 255 splitters; k_node_bucket drops
// every node into one of 256 buckets per order; k_node_rank counts, inside the bucket only, the keys below the
// node's own: position = bucket start + that count.  O(N * (log 256 + N/256)) instead of O(N^2).
struct NodeKey {
    int64_t v;
    uint32_t idx;
};
__device__ __forceinline__ bool key_less(int64_t av, uint32_t ai, int64_t bv, uint32_t bi) {
    return av < bv || (av == bv && ai < bi);
}
// KS_SCORE_LEAST_ALLOCATED bound: the score of node n for a pod that requests nothing.  For requests >= 0 the score of
// every feasible (pod, n) cell is <= least_alloc_bound(n) (same truncating divisions, monotone in the numerators).
__device__ __forceinline__ int64_t least_alloc_bound(const NodeTable& nt, uint32_t n) {
    return least_alloc_int(nt.free_cpu[n], nt.free_mem[n], nt.alloc_cpu[n], nt.alloc_mem[n], 0, 0);
}
// prio[0..Npad) = leftover priority, prio[Npad..Npad+N) = least-allocated bound (k_node_bound, once per build)
__device__ __forceinline__ int64_t order_value(const NodeTable& nt, const int64_t* __restrict__ prio, int k, uint32_t n) {
    return k == 0 ? nt.free_cpu[n] : (k == 1 ? nt.free_mem[n] : (k == 2 ? -prio[n] : -prio[(size_t)nt.Npad + n]));
}

// least-allocated bound of every node + which label bits some node carries (a selector naming a dead bit is
// infeasible everywhere: the argmax kernels answer it without scanning)
__global__ void __launch_bounds__(256) k_node_bound(NodeTable nt, int64_t* __restrict__ bound, unsigned long long* __restrict__ live) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nt.N) return;
    bound[n] = least_alloc_bound(nt, n);
    // [2]: max allocatable cpu, memory.  A node with allocatable <= 0 scores 0 for that resource whatever the request,
    // its bound too, so it gives k_least_alloc's per-pod slack nothing: it counts as INT64_MAX, which makes that term 0.
    long long* amax = reinterpret_cast<long long*>(live + KS_MAX_LABEL_WORDS);
    const long long ac = nt.alloc_cpu[n] > 0 ? nt.alloc_cpu[n] : INT64_MAX, am = nt.alloc_mem[n] > 0 ? nt.alloc_mem[n] : INT64_MAX;
    if (ac > __ldcg(amax)) atomicMax(amax, ac);
    if (am > __ldcg(amax + 1)) atomicMax(amax + 1, am);
    for (uint32_t w = 0; w < nt.W; w++) {
        const unsigned long long v = nt.labels[(size_t)w * nt.Npad + n];
        if (v & ~__ldcg(live + w)) atomicOr(live + w, v);
    }
}

constexpr int RANK_SAMPLES = 1024, RANK_BUCKETS = 256;
// Work cursors of k_mask_rows (one per column block), zeroed by k_pod_ranks.  One cursor per 128-byte line: with all cursors in one line the L2 serialised every claim of the whole chip on it
// (~3 ns each: 781k claims = the whole 2.4 ms the kernel then took at C3, whatever the block size).
constexpr uint32_t RW_CURSOR_STRIDE = 32;
// Splitters per resource in k_pod_ranks' shared memory (dynamic, 16 bytes per splitter pair: <= 128 KB).  With 8192 the part
// of a search that is left for the sorted array in L2 covers <= 7 elements of one 64-byte block (C3: stride 8): ~1.6 random
// 32-byte sector requests per search instead of ~4 with 2048 splitters - and that request rate is what bounds the kernel.
constexpr int RANK_SPLITTERS = 8192;
constexpr int RANK_THREADS = 1024; // one CTA per SM
constexpr int N_ORDERS = 4; // free_cpu, free_mem, leftover priority, least-allocated bound

__global__ void __launch_bounds__(RANK_SAMPLES)
    k_node_splitters(NodeTable nt, const int64_t* __restrict__ prio, int64_t* __restrict__ spl_v,
                     uint32_t* __restrict__ spl_i, uint32_t* __restrict__ hist) {
    __shared__ int64_t s_v[RANK_SAMPLES];
    __shared__ uint32_t s_i[RANK_SAMPLES];
    const uint32_t t = threadIdx.x, k = blockIdx.x; // one CTA per order
    const uint32_t n = (uint32_t)(((uint64_t)t * nt.N) / RANK_SAMPLES);
    s_v[t] = order_value(nt, prio, k, n);
    s_i[t] = n;
    if (t < RANK_BUCKETS) hist[k * RANK_BUCKETS + t] = 0;
    __syncthreads();
    for (uint32_t size = 2; size <= RANK_SAMPLES; size <<= 1)
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            if (t < RANK_SAMPLES / 2) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const int64_t av = s_v[lo], bv = s_v[hi];
                const uint32_t ai = s_i[lo], bi = s_i[hi];
                if (key_less(bv, bi, av, ai) == up) {
                    s_v[lo] = bv; s_i[lo] = bi;
                    s_v[hi] = av; s_i[hi] = ai;
                }
            }
            __syncthreads();
        }
    if (t < RANK_BUCKETS - 1) { // splitter j = sample 4(j+1)-1
        spl_v[k * RANK_BUCKETS + t] = s_v[4 * (t + 1) - 1];
        spl_i[k * RANK_BUCKETS + t] = s_i[4 * (t + 1) - 1];
    }
}

__global__ void __launch_bounds__(256)
    k_node_bucket(NodeTable nt, const int64_t* __restrict__ prio, const int64_t* __restrict__ spl_v,
                  const uint32_t* __restrict__ spl_i, uint32_t* __restrict__ hist, uint8_t* __restrict__ bkt,
                  uint32_t* __restrict__ loc) {
    __shared__ int64_t s_v[N_ORDERS][RANK_BUCKETS];
    __shared__ uint32_t s_i[N_ORDERS][RANK_BUCKETS];
    for (uint32_t j = threadIdx.x; j < N_ORDERS * (RANK_BUCKETS - 1); j += blockDim.x) {
        const uint32_t k = j / (RANK_BUCKETS - 1), q = j % (RANK_BUCKETS - 1);
        s_v[k][q] = spl_v[k * RANK_BUCKETS + q];
        s_i[k][q] = spl_i[k * RANK_BUCKETS + q];
    }
    __syncthreads();
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nt.N) return;
#pragma unroll
    for (int k = 0; k < N_ORDERS; k++) {
        const int64_t v = order_value(nt, prio, k, n);
        uint32_t lo = 0, len = RANK_BUCKETS - 1; // number of splitters < key
        while (len > 0) {
            const uint32_t half = len >> 1;
            if (key_less(s_v[k][lo + half], s_i[k][lo + half], v, n)) {
                lo += half + 1;
                len -= half + 1;
            } else {
                len = half;
            }
        }
        bkt[(size_t)k * nt.N + n] = (uint8_t)lo;
        loc[(size_t)k * nt.N + n] = atomicAdd(&hist[k * RANK_BUCKETS + lo], 1u);
    }
}

// bucket-ordered node lists (order inside a bucket is arbitrary; k_node_rank fixes the final positions)
__global__ void __launch_bounds__(256)
    k_node_scatter(uint32_t N, const uint32_t* __restrict__ hist, const uint8_t* __restrict__ bkt,
                   const uint32_t* __restrict__ loc, uint32_t* __restrict__ perm) {
    __shared__ uint32_t s_start[N_ORDERS][RANK_BUCKETS];
    if (threadIdx.x < N_ORDERS) {
        uint32_t acc = 0;
        for (int b = 0; b < RANK_BUCKETS; b++) {
            s_start[threadIdx.x][b] = acc;
            acc += hist[threadIdx.x * RANK_BUCKETS + b];
        }
    }
    __syncthreads();
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
#pragma unroll
    for (int k = 0; k < N_ORDERS; k++)
        perm[(size_t)k * N + s_start[k][bkt[(size_t)k * N + n]] + loc[(size_t)k * N + n]] = n;
}

__global__ void __launch_bounds__(256)
    k_node_rank(NodeTable nt, const int64_t* __restrict__ prio, const uint32_t* __restrict__ hist,
                const uint8_t* __restrict__ bkt, const uint32_t* __restrict__ perm, int64_t* __restrict__ sortedC,
                int64_t* __restrict__ sortedM, uint32_t* __restrict__ gposC, uint32_t* __restrict__ gposM,
                int64_t* __restrict__ ord_prio, int32_t* __restrict__ ord_idx, uint32_t Nord,
                int64_t* __restrict__ splC, int64_t* __restrict__ splM, uint32_t spl_stride,
                int64_t* __restrict__ ordL_s0, int32_t* __restrict__ ordL_idx) {
    __shared__ uint32_t s_start[N_ORDERS][RANK_BUCKETS + 1];
    if (threadIdx.x < N_ORDERS) {
        uint32_t acc = 0;
        for (int b = 0; b < RANK_BUCKETS; b++) {
            s_start[threadIdx.x][b] = acc;
            acc += hist[threadIdx.x * RANK_BUCKETS + b];
        }
        s_start[threadIdx.x][RANK_BUCKETS] = acc;
    }
    __syncthreads();
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t N = nt.N;
    if (n < N) {
        uint32_t pos[N_ORDERS];
#pragma unroll
        for (int k = 0; k < N_ORDERS; k++) {
            const int64_t v = order_value(nt, prio, k, n);
            const uint32_t b = bkt[(size_t)k * N + n];
            uint32_t c = 0;
            for (uint32_t j = s_start[k][b]; j < s_start[k][b + 1]; j++) {
                const uint32_t m = perm[(size_t)k * N + j];
                c += key_less(order_value(nt, prio, k, m), m, v, n);
            }
            pos[k] = s_start[k][b] + c;
        }
        const int64_t fc = nt.free_cpu[n], fm = nt.free_mem[n];
        gposC[n] = pos[0];
        gposM[n] = pos[1];
        sortedC[pos[0]] = fc;
        sortedM[pos[1]] = fm;
        if (pos[0] % spl_stride == 0) splC[pos[0] / spl_stride] = fc;
        if (pos[1] % spl_stride == 0) splM[pos[1] / spl_stride] = fm;
        ord_prio[pos[2]] = prio[n];
        ord_idx[pos[2]] = (int32_t)n;
        ordL_s0[pos[3]] = prio[(size_t)nt.Npad + n];
        ordL_idx[pos[3]] = (int32_t)n;
    } else if (n < Nord) { // padding of the priority / bound orders
        ord_prio[n] = INT64_MIN;
        ord_idx[n] = -1;
        ordL_s0[n] = INT64_MIN;
        ordL_idx[n] = -1;
    }
}

// One CTA builds tile k of an index in the column-block format (ks_bitpar.h): its prefix rows and label-pair columns, at
// 32 * (k % 8) of the 256-byte lines of column block k / 8.  slot_node maps the index's slots to nodes (nullptr = node
// order).  Optional outputs: tile_sorted (node order, for k_build_ranks) gets the tile's global positions in ascending
// order; bk (the ordered indexes, for the argmax kernels) gets the tile's column of the bucket arrays, which have no
// columns for the padding tiles.
__global__ void __launch_bounds__(288)
    k_build_tiles(NodeTable nt, const uint32_t* __restrict__ gposC, const uint32_t* __restrict__ gposM,
                  const int32_t* __restrict__ slot_node, uint8_t* __restrict__ blob, RowsLayout lay,
                  uint32_t* __restrict__ tile_sorted, TileBuckets bk) {
    __shared__ uint32_t s_g[2][BP_TILE];
    __shared__ uint16_t s_lr[2][BP_TILE];
    __shared__ uint8_t s_valid[BP_TILE];
    __shared__ uint64_t s_lab[KS_MAX_LABEL_WORDS][BP_TILE];
    const uint32_t tile_g = blockIdx.x, cb = tile_g / RW_TILES, t = tile_g % RW_TILES, s = threadIdx.x;
    const uint32_t n_tiles_pad = lay.ncb * RW_TILES;
    uint8_t* B = blob + (size_t)cb * lay.cb_stride;
    if (s < BP_TILE) {
        const uint32_t slot = tile_g * BP_TILE + s;
        const bool v = slot < nt.N;
        const uint32_t n = v ? (slot_node ? (uint32_t)slot_node[slot] : slot) : 0;
        s_valid[s] = v;
        s_g[0][s] = v ? gposC[n] : 0xFFFFFFFFu;
        s_g[1][s] = v ? gposM[n] : 0xFFFFFFFFu;
        for (uint32_t w = 0; w < nt.W; w++) s_lab[w][s] = v ? nt.labels[(size_t)w * nt.Npad + n] : 0ull;
    }
    __syncthreads();
    if (s < BP_TILE) {
        for (int r = 0; r < 2; r++) {
            const uint32_t g = s_g[r][s];
            uint32_t c = 0;
            for (int k = 0; k < BP_TILE; k++) c += s_g[r][k] < g;
            s_lr[r][s] = (uint16_t)c;
            // positions are distinct, so the valid slots fill tile_sorted[0..count) exactly; the rest is +inf
            if (tile_sorted) {
                uint32_t* ts = tile_sorted + ((size_t)r * n_tiles_pad + tile_g) * BP_TILE;
                if (s_valid[s]) ts[c] = g;
                const uint32_t count = nt.N > tile_g * BP_TILE ? min((uint32_t)BP_TILE, nt.N - tile_g * BP_TILE) : 0u;
                if (s >= count) ts[s] = 0xFFFFFFFFu;
            }
        }
    }
    __syncthreads();
    // prefix tables: row r = slots of the tile whose tile-local rank is >= r  (i.e. free >= threshold)
    if (s < BP_ROWS) {
        for (int r = 0; r < 2; r++) {
            uint32_t w[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                uint32_t acc = 0;
                for (int b = 0; b < 32; b++) {
                    const int k = j * 32 + b;
                    acc |= (uint32_t)(s_valid[k] && s_lr[r][k] >= s) << b;
                }
                w[j] = acc;
            }
            uint8_t* line = B + (r ? lay.off_tabM : lay.off_tabC) + (size_t)s * RW_LINE + t * 32;
            *reinterpret_cast<uint4*>(line) = make_uint4(w[0], w[1], w[2], w[3]);
            *reinterpret_cast<uint4*>(line + 16) = make_uint4(w[4], w[5], w[6], w[7]);
        }
    }
    // bucket membership + base counts of this tile's column
    if (bk.base[0] && tile_g < lay.n_tiles) {
        const uint32_t nb = (nt.N >> 6) + 1;
        for (uint32_t hi = s; hi < nb; hi += blockDim.x) {
            bk.memb[0][(size_t)hi * lay.n_tiles + tile_g] = 0ull;
            bk.memb[1][(size_t)hi * lay.n_tiles + tile_g] = 0ull;
        }
        __syncthreads();
        if (s < BP_TILE && s_valid[s]) {
            atomicOr(&bk.memb[0][(size_t)(s_g[0][s] >> 6) * lay.n_tiles + tile_g], 1ull << (s_g[0][s] & 63));
            atomicOr(&bk.memb[1][(size_t)(s_g[1][s] >> 6) * lay.n_tiles + tile_g], 1ull << (s_g[1][s] & 63));
        }
        __threadfence();
        __syncthreads();
        const uint32_t warp = s >> 5, lane = s & 31;
        if (warp < 2) {
            const unsigned long long* memb = warp ? bk.memb[1] : bk.memb[0];
            uint16_t* base = warp ? bk.base[1] : bk.base[0];
            uint32_t running = 0;
            for (uint32_t h0 = 0; h0 < nb; h0 += 32) {
                const uint32_t hi = h0 + lane;
                const uint32_t c = hi < nb ? __popcll(__ldcg(&memb[(size_t)hi * lay.n_tiles + tile_g])) : 0;
                uint32_t inc = c;
#pragma unroll
                for (int off = 1; off < 32; off <<= 1) {
                    const uint32_t o = __shfl_up_sync(0xffffffffu, inc, off);
                    if (lane >= (uint32_t)off) inc += o;
                }
                if (hi < nb) base[(size_t)hi * lay.n_tiles + tile_g] = (uint16_t)(running + inc - c);
                running += __shfl_sync(0xffffffffu, inc, 31);
            }
        }
    }
    // label-pair columns
    for (uint32_t bit = s; bit < 64u * nt.W; bit += blockDim.x) {
        const uint32_t w_ = bit >> 6, sh = bit & 63;
        uint32_t w[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            uint32_t acc = 0;
            for (int b = 0; b < 32; b++) acc |= (uint32_t)((s_lab[w_][j * 32 + b] >> sh) & 1ull) << b;
            w[j] = acc;
        }
        uint8_t* line = B + lay.off_pairs + (size_t)bit * RW_LINE + t * 32;
        *reinterpret_cast<uint4*>(line) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4*>(line + 16) = make_uint4(w[4], w[5], w[6], w[7]);
    }
}

// rank tables: the number of nodes of tile (cb, t) at sorted positions < g in a resource's order, for every threshold g in
// [0, N], as rank[cb][g][resource][j] u32 = tile j (low half) | tile j + 4 (high half), j < 4: the two tiles whose mask
// granules one lane of k_mask_rows writes.  One thread = one threshold of one column block: 8 binary searches per resource
// over the tiles' sorted positions (shared memory), one 16-byte store per resource.
__global__ void __launch_bounds__(256)
    k_build_ranks(const uint32_t* __restrict__ tile_sorted, RowsLayout lay, uint32_t* __restrict__ rank) {
    __shared__ uint32_t s_pos[2][RW_TILES][BP_TILE];
    const uint32_t cb = blockIdx.y, n_tiles_pad = lay.ncb * RW_TILES;
    for (uint32_t i = threadIdx.x; i < 2 * RW_TILES * BP_TILE; i += blockDim.x) {
        const uint32_t r = i / (RW_TILES * BP_TILE), tt = (i / BP_TILE) % RW_TILES, k = i % BP_TILE;
        s_pos[r][tt][k] = tile_sorted[((size_t)r * n_tiles_pad + cb * RW_TILES + tt) * BP_TILE + k];
    }
    __syncthreads();
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= lay.n_thr) return;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        uint32_t out[RW_TILES];
#pragma unroll
        for (uint32_t tt = 0; tt < RW_TILES; tt++) {
            const uint32_t* a = s_pos[r][tt];
            uint32_t lo = 0; // number of elements < g (0..256)
#pragma unroll
            for (uint32_t step = BP_TILE / 2; step > 0; step >>= 1)
                if (a[lo + step - 1] < g) lo += step;
            if (a[lo] < g) lo++; // lo <= 255 here
            out[tt] = lo;
        }
        uint32_t* dst = rank + (((size_t)cb * lay.n_thr + g) * 2 + r) * (RW_TILES / 2); // [cb][g][resource][tile pair]
        *reinterpret_cast<uint4*>(dst) = make_uint4(out[0] | (out[4] << 16), out[1] | (out[5] << 16),
                                                   out[2] | (out[6] << 16), out[3] | (out[7] << 16));
    }
}

// ------------------------------------------------------------------------------------------------ per call
template <class Ptr>
__device__ __forceinline__ uint32_t lower_bound_i64(Ptr a, uint32_t n, int64_t x) {
    uint32_t lo = 0, len = n; // number of elements < x
    while (len > 0) {
        const uint32_t half = len >> 1;
        if (a[lo + half] < x) {
            lo += half + 1;
            len -= half + 1;
        } else {
            len = half;
        }
    }
    return lo;
}

// rank = number of nodes with free < request; nodes at sorted positions >= rank satisfy request <= free
// (predicates.rs:42).  Two-level search: <=2048 splitters per resource in shared memory, then a window of
// spl_stride-1 elements of the global sorted array.
// The same kernel writes the mask kernel's pod records (thresholds, pod index, selector columns) in pod order: round 1
// sorted the pods by threshold to tame shared-memory bank conflicts; the rows format is conflict-free for any order and
// needs no sort.
constexpr uint32_t RW_SEL_GENERIC = 0xFFFFFFFFu;
constexpr uint32_t RW_PID_NONE = 0xFFFFFFFFu;

// the selector of a pod as record word: up to three required label-pair bit indices (10 bits each) + their number in
// bits 30-31; RW_SEL_GENERIC when it names more than three pairs (the mask kernel then walks the selector words)
template <class LoadWord>
__device__ __forceinline__ uint32_t selector_record(uint32_t W, LoadWord word) {
    uint32_t cols = 0, n_req = 0;
    for (uint32_t w = 0; w < W; w++) {
        unsigned long long bits = word(w);
        while (bits) { // required (key,value) pairs of the selector (predicates.rs:48)
            const uint32_t bit = w * 64 + __ffsll((long long)bits) - 1;
            bits &= bits - 1;
            if (n_req < 3) cols |= bit << (10 * n_req);
            n_req++;
        }
    }
    return n_req > 3 ? RW_SEL_GENERIC : (cols | (n_req << 30));
}

__global__ void __launch_bounds__(RANK_THREADS, 1)
    k_pod_ranks(PodView pv, const int64_t* __restrict__ sortedC, const int64_t* __restrict__ sortedM, uint32_t N,
                const int64_t* __restrict__ splC, const int64_t* __restrict__ splM, uint32_t n_spl, uint32_t stride,
                uint2* __restrict__ rk, uint32_t* __restrict__ cnt_zero, uint32_t W, uint4* __restrict__ rec,
                uint32_t* __restrict__ cursor, uint32_t n_cursor) {
    extern __shared__ __align__(16) unsigned char ranks_smem[];
    int64_t* const s_spl[2] = {reinterpret_cast<int64_t*>(ranks_smem), reinterpret_cast<int64_t*>(ranks_smem) + n_spl};
    if (threadIdx.x == 0) trace_start(TR_RANKS_START);
    if (blockIdx.x == 0) // the mask kernel's chunk cursors
        for (uint32_t k = threadIdx.x; k < n_cursor; k += blockDim.x) cursor[(size_t)k * RW_CURSOR_STRIDE] = 0;
    for (uint32_t k = threadIdx.x; k < n_spl; k += blockDim.x) {
        s_spl[0][k] = splC[k];
        s_spl[1][k] = splM[k];
    }
    __syncthreads();
    if (rec) // padding of the last group of 8
        for (uint32_t p = pv.P + blockIdx.x * blockDim.x + threadIdx.x; p < ((pv.P + 7u) & ~7u); p += gridDim.x * blockDim.x)
            rec[p] = make_uint4(0, 0, RW_PID_NONE, 0);
    // Two pods per thread and pass, i.e. four searches (2 pods x 2 resources) side by side: the part over the sorted array
    // in global memory is a chain of dependent L2 loads, and the four chains advance in lockstep (4 loads in flight).
    const uint32_t T = gridDim.x * blockDim.x;
    for (uint32_t p0 = blockIdx.x * blockDim.x + threadIdx.x; p0 < pv.P; p0 += 2 * T) {
        int64_t x[4];
        uint32_t lo[4], len[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { // k = 2 * pod + resource; a missing second pod searches for "below everything": no probes
            const uint32_t p = p0 + (k >> 1) * T;
            x[k] = p >= pv.P ? INT64_MIN : (k & 1) ? __ldg(pv.req_mem + p) : __ldg(pv.req_cpu + p);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t c = lower_bound_i64(s_spl[k & 1], n_spl, x[k]);
            lo[k] = c > 0 ? (c - 1) * stride + 1 : 0u; // sorted[lo-1] < x <= sorted[c*stride] (if it exists)
            len[k] = c > 0 ? min(stride - 1, N - lo[k]) : 0u;
        }
        while (len[0] | len[1] | len[2] | len[3]) {
            int64_t v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int64_t* sorted = (k & 1) ? sortedM : sortedC;
                v[k] = len[k] ? __ldg(sorted + lo[k] + (len[k] >> 1)) : 0;
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t half = len[k] >> 1;
                if (len[k] == 0) continue;
                if (v[k] < x[k]) {
                    lo[k] += half + 1;
                    len[k] -= half + 1;
                } else {
                    len[k] = half;
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const uint32_t p = p0 + q * T;
            if (p >= pv.P) break;
            rk[p] = make_uint2(lo[2 * q], lo[2 * q + 1]);
            if (cnt_zero) cnt_zero[p] = 0; // k_mask_rows accumulates feasible counts with REDs
            if (rec) // the mask kernel's 16-byte pod record, in pod order
                rec[p] = make_uint4(lo[2 * q], lo[2 * q + 1], p,
                                    selector_record(W, [&](uint32_t w) { return __ldg(pv.sel + (size_t)p * W + w); }));
        }
    }
    if (c_trace) {
        __syncthreads();
        if (threadIdx.x == 0) trace_end(TR_RANKS_END);
    }
}

// ------------------------------------------------------------------------------------------------ rows kernel
// k_mask_rows: the round-2 mask / count kernel ("rows" format, ks_bitpar.h).
//   * lane = (pod slot, t): 8 lanes per pod = 256 contiguous bytes of the pod's mask row; lane t stores granule t
//     (half of tile t/2) and granule 8 + t (half of tile 4 + t/2), so each of the two 128-bit store instructions
//     writes one whole 128-byte line per pod (on the H100, stores that leave every sector half-written run at half
//     the rate: BASELINE.md); a warp iteration covers 8 consecutive pods (two per thread, two independent chains);
//   * the tile-local ranks of the pod's thresholds come from the rank tables (one 32-bit load per resource from
//     L1/L2 = the ranks of the lane's two tiles; the 8 lanes of a pod read 16 contiguous bytes) - no
//     base/membership lookup, no POPC for ranks;
//   * table rows and label-pair columns are 256-byte lines in tile order: the 8 lanes of a shared-memory phase read
//     offsets 16 t (mod 128) of their own rows -> conflict-free for any ranks;
//   * work = (column block, pod group) items handed out dynamically: one atomic cursor per column block, each CTA claims
//     chunks of groups, a CTA whose block is exhausted re-stages the blob of the block with the most work left
//     (all SMs busy whatever ncb is, and SMs that stream faster simply claim more);
//   * pod records (pod order: no sort) arrive in a shared-memory ring by bulk copies a chunk ahead, and every warp loads
//     the rank entries of its next group before it stores the current one: under a saturated store stream the L2 load
//     replies queue behind the stores, and record and rank loads issued one group ahead left the stores waiting.
// k_count_rows: the same items without a mask (feasible counts only), claimed per warp with the records loaded one
// group ahead.  With no stores to hide them, the ring's chunk edges cost more than they save: at c3 the ring loop took
// 1.42 ms for the counts alone where this one takes 1.05 ms (H100, BASELINE.md §4).
__device__ __forceinline__ uint4 lds128(uint32_t a) { // pure: scheduled freely; ordered after the blob wait by the
    uint4 v;                                          // address dependence on the post-wait token
    asm("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ uint4 ldg128_keep(const uint4* p, uint64_t pol) { // L2 evict-last: pod records, read once per column block
    uint4 v;
    asm("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ uint32_t ldg_u32_keep(const uint32_t* p, uint64_t pol) { // L2 evict-last: the rank tables are re-read
    uint32_t v;
    asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}
template <class T>
__device__ __forceinline__ T* opaque_ptr(T* p) { // keeps a per-thread base pointer in one register pair (the compiler
    asm("" : "+l"(p));                           // would otherwise re-derive its lane part in every iteration)
    return p;
}
__device__ __forceinline__ uint4 and4(uint4 a, uint4 b) { return make_uint4(a.x & b.x, a.y & b.y, a.z & b.z, a.w & b.w); }
__device__ __forceinline__ uint4 and4(uint4 a, uint4 b, uint4 c) {
    return make_uint4(a.x & b.x & c.x, a.y & b.y & c.y, a.z & b.z & c.z, a.w & b.w & c.w);
}
struct RowsParams { // kernel parameters stay in the constant bank: the loop reads them from there on demand
    const uint8_t* blob;
    RowsLayout lay;
    const uint32_t* rank;            // [cb][threshold g][resource][j] = tile j | tile j + 4 << 16: 32 bytes per (cb, g)
    const uint4* rec_s;              // sorted pod records, padded to a multiple of 8
    const unsigned long long* sel_s; // the pods' selector words, pod order (generic path only)
    uint32_t n_groups;               // groups of 8 pods
    uint32_t* mask;                  // may be nullptr
    uint32_t row_words;              // mask row pitch in 32-bit words
    uint32_t* cnt;                   // may be nullptr
    uint32_t* cursor;                // [ncb * RW_CURSOR_STRIDE] next unclaimed pod group of every column block
    uint32_t chunk;                  // k_mask_rows: pod groups per ring slot, RW_CHUNK_MIN..RW_CHUNK_MAX (rows_chunk)
};
constexpr uint32_t RW_RING = 2; // record ring slots: a chunk is read while the next one is copied in
// Groups per chunk, measured at c3 on an H100 (BASELINE.md §4): 16-32 are equally fast, 64 gives back a third of the gain,
// and at 12 or fewer a chunk is over before the next one has landed.  The ring of 2 x 32 groups is 8 KB beside the blob.
constexpr uint32_t RW_CHUNK_MIN = 24, RW_CHUNK_MAX = 32;
constexpr uint32_t RW_CLAIM = 4; // k_count_rows: pod groups per claim (one atomicAdd per warp)
constexpr uint32_t RW_HOP_MIN = 256; // a partly claimed column block is worth moving to while it has this many groups left

// one lane's share of a (pod, column block) item: granules t (tile t/2) and 8 + t (tile 4 + t/2) of the pod's 256 bytes ->
// mask words a, b (128 cells); returns the number of feasible cells among them.
// a_tab = shared-window address of granule t of line 0 of tabC; tabM and the pair columns sit at constant offsets.
// rC, rM = tile-local ranks of the two tiles (low half: tile t/2, high half: tile 4 + t/2).
template <int W, bool PSMEM>
__device__ __forceinline__ uint32_t rows_item(const RowsParams& prm, uint32_t a_tab, uint32_t cb, uint32_t t, uint32_t* mask_col,
                                              bool st_hi, uint32_t rC, uint32_t rM, uint32_t pid, uint32_t sel, uint32_t q,
                                              uint64_t pol_st) {
    const uint32_t aC = a_tab + (rC & 0xFFFFu) * RW_LINE, aM = a_tab + RW_TAB_BYTES + (rM & 0xFFFFu) * RW_LINE;
    const uint32_t aC1 = a_tab + 128 + (rC >> 16) * RW_LINE, aM1 = a_tab + RW_TAB_BYTES + 128 + (rM >> 16) * RW_LINE;
    const uint4 c0 = lds128(aC), c1 = lds128(aC1);
    const uint4 m0 = lds128(aM), m1 = lds128(aM1);
    uint4 a, b;
    auto column = [&](uint32_t bit, uint4& q0, uint4& q1) { // node column of one required pair (predicates.rs:48-53)
        if (PSMEM) {
            const uint32_t ap = a_tab + bit * RW_LINE;
            q0 = lds128(ap + 2 * RW_TAB_BYTES);
            q1 = lds128(ap + 2 * RW_TAB_BYTES + 128);
        } else {
            const uint4* gp = reinterpret_cast<const uint4*>(prm.blob + (size_t)cb * prm.lay.cb_stride + prm.lay.off_pairs +
                                                             (size_t)bit * RW_LINE + t * 16u);
            q0 = __ldg(gp);
            q1 = __ldg(gp + 8);
        }
    };
    const uint32_t n_req = sel >> 30;
    if (n_req == 0) {
        a = and4(c0, m0);
        b = and4(c1, m1);
    } else if (sel != RW_SEL_GENERIC) {
        uint4 q0, q1;
        column(sel & 0x3FFu, q0, q1);
        a = and4(c0, m0, q0);
        b = and4(c1, m1, q1);
        if (n_req >= 2) {
            column((sel >> 10) & 0x3FFu, q0, q1);
            a = and4(a, q0);
            b = and4(b, q1);
            if (n_req == 3) {
                column((sel >> 20) & 0x3FFu, q0, q1);
                a = and4(a, q0);
                b = and4(b, q1);
            }
        }
    } else { // rare: more than three required pairs
        a = and4(c0, m0);
        b = and4(c1, m1);
#pragma unroll
        for (int w = 0; w < W; w++) {
            unsigned long long bits = __ldg(prm.sel_s + (size_t)q * W + w);
            while (bits) {
                const uint32_t bit = w * 64 + __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                uint4 q0, q1;
                column(bit, q0, q1);
                a = and4(a, q0);
                b = and4(b, q1);
            }
        }
    }
    if (mask_col != nullptr && pid != RW_PID_NONE) {
        uint32_t* dst = mask_col + (size_t)pid * prm.row_words; // granule t of the pod's 256-byte block
        // the mask is write-once streaming data: first in line for eviction from L2.  sm_90 stores at most 128 bits
        // per instruction; the 8 lanes of a pod store granules 0..7, then 8..15, so each instruction writes one whole
        // 128-byte line per pod.
        asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(dst), "r"(a.x), "r"(a.y), "r"(a.z),
                     "r"(a.w), "l"(pol_st)
                     : "memory");
        if (st_hi)
            asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(dst + 32), "r"(b.x), "r"(b.y),
                         "r"(b.z), "r"(b.w), "l"(pol_st)
                         : "memory");
    }
    return __popc(a.x) + __popc(a.y) + __popc(a.z) + __popc(a.w) + __popc(b.x) + __popc(b.y) + __popc(b.z) + __popc(b.w);
}

// (launch bounds of 1024 threads for both block sizes: 64 registers per thread, so that a 768-thread CTA leaves a quarter
// of the register file to the argmax CTAs that run beside it)
template <int W, bool PSMEM, int THREADS>
__global__ void __launch_bounds__(BP_THREADS, 1) k_mask_rows(const __grid_constant__ RowsParams prm) {
    extern __shared__ __align__(128) uint8_t smem[]; // the column block's blob, then the record ring
    __shared__ __align__(8) uint64_t bar;
    __shared__ __align__(8) uint64_t full[RW_RING], empty[RW_RING];
    __shared__ uint32_t s_base[RW_RING];
    __shared__ unsigned long long s_key;
    constexpr uint32_t WARPS = THREADS / 32;
    const uint32_t tid = threadIdx.x, t = tid & 7, ps = (tid >> 3) & 3, lane = tid & 31, warp = tid >> 5;
    uint64_t pol_st, pol_ld; // L2 policies: mask stores evict-first, rank-table and pod-record loads evict-last
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_st));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_ld));
    if (tid == 0) {
        mbar_init(&bar, 1);
        for (uint32_t s = 0; s < RW_RING; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WARPS);
        }
        fence_mbar_init();
        trace_start(TR_MASK_START);
    }
    __syncthreads();
    uint32_t phase = 0;

    // Work = (column block, pod group) items.  Every column block has one cursor (zeroed by k_pod_ranks); thread 0 claims
    // C = prm.chunk consecutive pod groups of the staged column block at a time with one atomicAdd, one chunk ahead of
    // their use, and brings the chunk's records (C x 128 contiguous bytes) into a ring slot in shared memory by a bulk
    // copy while the warps work on the chunk before.  The CTA's chunks are numbered across column blocks (slot x % RW_RING
    // holds chunk x; full[s] completes when its records have landed, empty[s] when every warp is done reading them), and
    // their groups are dealt to the warps round robin.  A chunk whose base lies past the block's end closes the block.
    // The CTAs that share a column block therefore finish it together whatever their individual rates (SMs do not all
    // stream at the same rate), and a CTA whose block is exhausted moves - one barrier, one re-staging of the blob - to
    // the block with the most unclaimed groups.  CTAs start spread evenly over the column blocks.
    const uint32_t n_slots = prm.n_groups; // pod groups per column block
    const uint32_t ncb = prm.lay.ncb;
    const uint32_t C = prm.chunk;
    uint8_t* const ring = smem + prm.lay.smem_bytes;
    uint32_t seq = 0;       // chunks begun by this CTA
    uint32_t pending = 0;   // thread 0: the claim for the next chunk
    bool prod_done = false; // thread 0: the block's closing chunk has been issued
    uint32_t cb = (uint32_t)((uint64_t)blockIdx.x * ncb / gridDim.x);
    for (;;) { // one iteration per column block this CTA works on
        __syncthreads(); // all reads of the previous blob are done
        uint32_t* cursor = prm.cursor + (size_t)cb * RW_CURSOR_STRIDE;
        auto issue = [&](uint32_t x) { // thread 0: claimed chunk -> ring slot x % RW_RING, once its previous chunk is read
            const uint32_t s = x % RW_RING;
            mbar_wait(&empty[s], ((x / RW_RING) & 1u) ^ 1u);
            const uint32_t b = pending;
            s_base[s] = b;
            if (b < n_slots) {
                const uint32_t bytes = min(C, n_slots - b) * 128u;
                fence_proxy_async();
                mbar_arrive_expect_tx(&full[s], bytes);
                tma_bulk_g2s(ring + (size_t)s * C * 128u, prm.rec_s + (size_t)b * 8u, bytes, &full[s], pol_ld);
                pending = atomicAdd(cursor, C);
            } else {
                mbar_arrive(&full[s]);
                prod_done = true;
            }
        };
        if (tid == 0) {
            fence_proxy_async();
            mbar_arrive_expect_tx(&bar, prm.lay.smem_bytes);
            const uint8_t* src = prm.blob + (size_t)cb * prm.lay.cb_stride;
            for (uint32_t off = 0; off < prm.lay.smem_bytes; off += 32768u)
                tma_bulk_g2s(smem + off, src + off, min(32768u, prm.lay.smem_bytes - off), &bar);
            pending = atomicAdd(cursor, C);
            prod_done = false;
            issue(seq);
        }
        // rank entry of (g, resource r, tiles t/2 and 4 + t/2): rk_t[g * 8 + r * 4]
        const uint32_t* rk_t = opaque_ptr(prm.rank + (size_t)cb * prm.lay.n_thr * RW_TILES + (t >> 1));
        auto fetch_ranks = [&](const uint4& ra, const uint4& rb, uint32_t& rCa, uint32_t& rMa, uint32_t& rCb, uint32_t& rMb) {
            rCa = ldg_u32_keep(rk_t + (size_t)ra.x * 8u, pol_ld);
            rMa = ldg_u32_keep(rk_t + (size_t)ra.y * 8u + 4, pol_ld);
            rCb = ldg_u32_keep(rk_t + (size_t)rb.x * 8u, pol_ld);
            rMb = ldg_u32_keep(rk_t + (size_t)rb.y * 8u + 4, pol_ld);
        };
        // this warp's next group: index i of chunk j (warp-uniform), whose first group is base and which holds cnt groups
        uint32_t j = seq, i = warp, base = 0, cnt = 0;
        auto enter = [&]() {
            if (tid == 0 && !prod_done) issue(j + 1);
            mbar_wait(&full[j % RW_RING], (j / RW_RING) & 1u);
            base = s_base[j % RW_RING];
            cnt = base < n_slots ? min(C, n_slots - base) : 0u;
        };
        auto settle = [&]() { // moves (j, i) on to this warp's next group; false at the block's closing chunk
            while (i >= cnt && cnt != 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[j % RW_RING]);
                i = i >= C ? i - C : 0u; // (a chunk cut short by the block's end is followed by the closing chunk)
                j++;
                enter();
            }
            return cnt != 0;
        };
        auto rec = [&](uint32_t q) { // record of pod 2 ps + q of the group
            return *reinterpret_cast<const uint4*>(ring + ((size_t)(j % RW_RING) * C + i) * 128u + (2u * ps + q) * 16u);
        };
        enter();
        bool more = settle();
        uint4 nA = make_uint4(0, 0, RW_PID_NONE, 0), nB = nA;
        uint32_t nCa = 0, nMa = 0, nCb = 0, nMb = 0;
        if (more) {
            nA = rec(0);
            nB = rec(1);
            fetch_ranks(nA, nB, nCa, nMa, nCb, nMb);
        }

        mbar_wait(&bar, phase);
        phase ^= 1;
        uint32_t tok; // every shared-memory load below depends on a value produced after the wait
        asm volatile("mov.u32 %0, 0;" : "=r"(tok)::"memory");
        const uint32_t a_tab = smem_u32(smem) + t * 16u + tok;
        // a tile is written when it holds nodes, or when the caller's row pitch has room for it (a pitch that is a multiple
        // of 256 bytes - ks_mask_row_bytes_aligned - lets the 8 lanes of a pod always store one whole, 256-byte-aligned
        // block: two whole 128-byte lines); padding tiles hold zeros.  This lane writes half of tile t/2 and half of
        // tile 4 + t/2; the condition falls with the tile index, so st_hi implies that the low granule is written too.
        auto written = [&](uint32_t tile) { return tile < prm.lay.n_tiles || (tile + 1u) * 8u <= prm.row_words; };
        const uint32_t tile_lo = cb * RW_TILES + (t >> 1);
        const bool st_hi = written(tile_lo + 4);
        uint32_t* mask_col = (prm.mask != nullptr && written(tile_lo))
                                 ? opaque_ptr(prm.mask + (size_t)cb * (RW_LINE / 4) + t * 4u)
                                 : nullptr;

        while (more) { // warp-uniform: one pod group; the next group's records and ranks are loaded before its stores
            const uint32_t pidA = nA.z, selA = nA.w, pidB = nB.z, selB = nB.w;
            const uint32_t rCa = nCa, rMa = nMa, rCb = nCb, rMb = nMb;
            const uint32_t g = base + i;
            i += WARPS;
            more = settle();
            if (more) {
                nA = rec(0);
                nB = rec(1);
                fetch_ranks(nA, nB, nCa, nMa, nCb, nMb);
            }
            const uint32_t cA = rows_item<W, PSMEM>(prm, a_tab, cb, t, mask_col, st_hi, rCa, rMa, pidA, selA, g * 8u + 2u * ps, pol_st);
            const uint32_t cB = rows_item<W, PSMEM>(prm, a_tab, cb, t, mask_col, st_hi, rCb, rMb, pidB, selB, g * 8u + 2u * ps + 1u, pol_st);
            if (prm.cnt != nullptr) { // the 8 lanes of a pod are adjacent; both pods' counts ride in one register
                uint32_t c = cA | (cB << 16);
                c += __shfl_xor_sync(0xffffffffu, c, 1);
                c += __shfl_xor_sync(0xffffffffu, c, 2);
                c += __shfl_xor_sync(0xffffffffu, c, 4);
                if (t == 0) {
                    const uint32_t ca = c & 0xFFFFu, cb_ = c >> 16;
                    if (ncb == 1) { // single writer, no zero-init needed
                        if (pidA != RW_PID_NONE) prm.cnt[pidA] = ca;
                        if (pidB != RW_PID_NONE) prm.cnt[pidB] = cb_;
                    } else {
                        if (pidA != RW_PID_NONE && ca) atomicAdd(&prm.cnt[pidA], ca);
                        if (pidB != RW_PID_NONE && cb_) atomicAdd(&prm.cnt[pidB], cb_);
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[j % RW_RING]); // the closing chunk
        seq = j + 1;

        // this column block is exhausted (its last groups are being finished by the warps that claimed them, here or in
        // other CTAs): move to the block with the most unclaimed groups, if any is worth a re-staging
        if (ncb == 1) break;
        __syncthreads();
        if (tid == 0) s_key = 0;
        __syncthreads();
        for (uint32_t c = tid; c < ncb; c += THREADS) {
            const uint32_t used = *reinterpret_cast<volatile uint32_t*>(prm.cursor + (size_t)c * RW_CURSOR_STRIDE);
            const uint32_t left = used < n_slots ? n_slots - used : 0u;
            if (left >= RW_HOP_MIN || (left > 0 && used == 0)) { // key: groups left, then nearness to the current block
                const uint32_t dist = (c + ncb - cb) % ncb;
                atomicMax(&s_key, ((unsigned long long)left << 32) | (0xFFFFFFFFu - dist));
            }
        }
        __syncthreads();
        const unsigned long long key = s_key;
        if (key == 0) break;
        cb = (cb + (0xFFFFFFFFu - (uint32_t)key)) % ncb;
    }
    if (c_trace) {
        __syncthreads();
        if (tid == 0) {
            const unsigned long long now = global_ns();
            atomicMax(c_trace + TR_MASK_END, now);
            atomicMax(c_trace + TR_MASK_FIRST_CTA_END_INV, ~now); // = ~(earliest CTA end)
        }
    }
}

template <int W, bool PSMEM, int THREADS>
__global__ void __launch_bounds__(BP_THREADS, 1) k_count_rows(const __grid_constant__ RowsParams prm) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ unsigned long long s_key;
    const uint32_t tid = threadIdx.x, t = tid & 7, ps = (tid >> 3) & 3;
    uint64_t pol_st, pol_ld; // L2 policies: mask stores evict-first, rank-table and pod-record loads evict-last
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_st));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_ld));
    if (tid == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
        trace_start(TR_MASK_START);
    }
    __syncthreads();
    uint32_t phase = 0;

    // Work = (column block, pod group) items.  Every column block has one cursor (zeroed by k_pod_ranks); a warp claims
    // RW_CLAIM consecutive pod groups of the staged column block at a time with one atomicAdd, one claim ahead of the one
    // it is working on.  The CTAs that share a column block therefore finish it together whatever their individual rates
    // (SMs do not all stream at the same rate), and a CTA whose block is exhausted moves - one barrier, one re-staging of the 148 KB blob - to the block
    // with the most unclaimed groups.  CTAs start spread evenly over the column blocks.
    const uint32_t n_slots = prm.n_groups; // pod groups per column block
    const uint32_t ncb = prm.lay.ncb;
    const uint32_t lane = tid & 31;
    const uint32_t last_grp = n_slots - 1;
    const uint4* rec_t = opaque_ptr(prm.rec_s + 2 * ps); // this thread's pods: 2*ps and 2*ps+1 of the group (neighbours)
    // loads are unconditional (group index clamped into the list)
    auto fetch_rec = [&](uint32_t j, uint4& ra, uint4& rb) {
        const uint4* rp = rec_t + (size_t)min(j, last_grp) * 8u;
        ra = ldg128_keep(rp, pol_ld);
        rb = ldg128_keep(rp + 1, pol_ld);
    };
    uint32_t cb = (uint32_t)((uint64_t)blockIdx.x * ncb / gridDim.x);
    for (;;) { // one iteration per column block this CTA works on
        __syncthreads(); // all reads of the previous blob are done
        if (tid == 0) {
            fence_proxy_async();
            mbar_arrive_expect_tx(&bar, prm.lay.smem_bytes);
            const uint8_t* src = prm.blob + (size_t)cb * prm.lay.cb_stride;
            for (uint32_t off = 0; off < prm.lay.smem_bytes; off += 32768u)
                tma_bulk_g2s(smem + off, src + off, min(32768u, prm.lay.smem_bytes - off), &bar);
        }
        uint32_t* cursor = prm.cursor + (size_t)cb * RW_CURSOR_STRIDE;
        auto claim = [&]() -> uint32_t { // lane 0 holds the result; broadcast where it is needed
            return lane == 0 ? atomicAdd(cursor, RW_CLAIM) : 0u;
        };
        uint32_t base = __shfl_sync(0xffffffffu, claim(), 0);
        uint32_t next_raw = claim();
        // rank entry of (g, resource r, tiles t/2 and 4 + t/2): rk_t[g * 8 + r * 4]
        const uint32_t* rk_t = opaque_ptr(prm.rank + (size_t)cb * prm.lay.n_thr * RW_TILES + (t >> 1));
        auto fetch_ranks = [&](const uint4& ra, const uint4& rb, uint32_t& rCa, uint32_t& rMa, uint32_t& rCb, uint32_t& rMb) {
            rCa = ldg_u32_keep(rk_t + (size_t)ra.x * 8u, pol_ld);
            rMa = ldg_u32_keep(rk_t + (size_t)ra.y * 8u + 4, pol_ld);
            rCb = ldg_u32_keep(rk_t + (size_t)rb.x * 8u, pol_ld);
            rMb = ldg_u32_keep(rk_t + (size_t)rb.y * 8u + 4, pol_ld);
        };
        // records of iteration k+1 are in flight while k computes (its ranks are loaded at the top of k; a deeper pipeline
        // - records two ahead, ranks one ahead - has not been tried on the H100)
        uint4 nA, nB;
        fetch_rec(base, nA, nB);

        mbar_wait(&bar, phase);
        phase ^= 1;
        uint32_t tok; // every shared-memory load below depends on a value produced after the wait
        asm volatile("mov.u32 %0, 0;" : "=r"(tok)::"memory");
        const uint32_t a_tab = smem_u32(smem) + t * 16u + tok;
        // a tile is written when it holds nodes, or when the caller's row pitch has room for it (a pitch that is a multiple
        // of 256 bytes - ks_mask_row_bytes_aligned - lets the 8 lanes of a pod always store one whole, 256-byte-aligned
        // block: two whole 128-byte lines); padding tiles hold zeros.  This lane writes half of tile t/2 and half of
        // tile 4 + t/2; the condition falls with the tile index, so st_hi implies that the low granule is written too.
        auto written = [&](uint32_t tile) { return tile < prm.lay.n_tiles || (tile + 1u) * 8u <= prm.row_words; };
        const uint32_t tile_lo = cb * RW_TILES + (t >> 1);
        const bool st_hi = written(tile_lo + 4);
        uint32_t* mask_col = (prm.mask != nullptr && written(tile_lo))
                                 ? opaque_ptr(prm.mask + (size_t)cb * (RW_LINE / 4) + t * 4u)
                                 : nullptr;

        while (base < n_slots) { // warp-uniform: one claim of up to RW_CLAIM pod groups
            const uint32_t end = min(base + RW_CLAIM, n_slots);
            uint32_t next = 0;
            for (uint32_t j = base; j < end; j++) {
                const uint32_t pidA = nA.z, selA = nA.w, pidB = nB.z, selB = nB.w;
                uint32_t rCa, rMa, rCb, rMb;
                fetch_ranks(nA, nB, rCa, rMa, rCb, rMb);
                uint32_t jn = j + 1;
                if (jn == end) { // last group of the claim: the next claim (requested a whole claim ago) says what follows
                    next = __shfl_sync(0xffffffffu, next_raw, 0);
                    jn = next;
                }
                fetch_rec(jn, nA, nB);
                const uint32_t cA = rows_item<W, PSMEM>(prm, a_tab, cb, t, mask_col, st_hi, rCa, rMa, pidA, selA, j * 8u + 2u * ps, pol_st);
                const uint32_t cB = rows_item<W, PSMEM>(prm, a_tab, cb, t, mask_col, st_hi, rCb, rMb, pidB, selB, j * 8u + 2u * ps + 1u, pol_st);
                if (prm.cnt != nullptr) { // the 8 lanes of a pod are adjacent; both pods' counts ride in one register
                    uint32_t c = cA | (cB << 16);
                    c += __shfl_xor_sync(0xffffffffu, c, 1);
                    c += __shfl_xor_sync(0xffffffffu, c, 2);
                    c += __shfl_xor_sync(0xffffffffu, c, 4);
                    if (t == 0) {
                        const uint32_t ca = c & 0xFFFFu, cb_ = c >> 16;
                        if (ncb == 1) { // single writer, no zero-init needed
                            if (pidA != RW_PID_NONE) prm.cnt[pidA] = ca;
                            if (pidB != RW_PID_NONE) prm.cnt[pidB] = cb_;
                        } else {
                            if (pidA != RW_PID_NONE && ca) atomicAdd(&prm.cnt[pidA], ca);
                            if (pidB != RW_PID_NONE && cb_) atomicAdd(&prm.cnt[pidB], cb_);
                        }
                    }
                }
            }
            base = next;
            if (base < n_slots) next_raw = claim();
        }

        // this column block is exhausted (its last groups are being finished by the warps that claimed them, here or in
        // other CTAs): move to the block with the most unclaimed groups, if any is worth a re-staging
        if (ncb == 1) break;
        __syncthreads();
        if (tid == 0) s_key = 0;
        __syncthreads();
        for (uint32_t c = tid; c < ncb; c += THREADS) {
            const uint32_t used = *reinterpret_cast<volatile uint32_t*>(prm.cursor + (size_t)c * RW_CURSOR_STRIDE);
            const uint32_t left = used < n_slots ? n_slots - used : 0u;
            if (left >= RW_HOP_MIN || (left > 0 && used == 0)) { // key: groups left, then nearness to the current block
                const uint32_t dist = (c + ncb - cb) % ncb;
                atomicMax(&s_key, ((unsigned long long)left << 32) | (0xFFFFFFFFu - dist));
            }
        }
        __syncthreads();
        const unsigned long long key = s_key;
        if (key == 0) break;
        cb = (cb + (0xFFFFFFFFu - (uint32_t)key)) % ncb;
    }
    if (c_trace) {
        __syncthreads();
        if (tid == 0) {
            const unsigned long long now = global_ns();
            atomicMax(c_trace + TR_MASK_END, now);
            atomicMax(c_trace + TR_MASK_FIRST_CTA_END_INV, ~now); // = ~(earliest CTA end)
        }
    }
}

// ---- argmax of the separable score = first feasible node in descending priority order ----
// The priority-ordered index (blobP) is read through L1/L2.  Phase 1 (k_first_fit_head): one thread per pod
// looks at the two best tiles (512 best nodes) - enough for almost every pod; the rest is appended to a list.
// Phase 2 (k_first_fit_tail): one warp per listed pod, one tile per lane, 32 tiles per step, ballot + early exit.
struct PodThreshold {
    const uint16_t* baseC;
    const uint16_t* baseM;
    const unsigned long long* membC;
    const unsigned long long* membM;
    unsigned long long lowC, lowM;
};

// tile-local ranks through the bucket arrays of the index's order (TileBuckets, ks_bitpar.h)
__device__ __forceinline__ PodThreshold pod_threshold(const TileBuckets& bk, const RowsLayout& lay, uint2 r) {
    PodThreshold t;
    t.baseC = bk.base[0] + (size_t)(r.x >> 6) * lay.n_tiles;
    t.baseM = bk.base[1] + (size_t)(r.y >> 6) * lay.n_tiles;
    t.membC = bk.memb[0] + (size_t)(r.x >> 6) * lay.n_tiles;
    t.membM = bk.memb[1] + (size_t)(r.y >> 6) * lay.n_tiles;
    t.lowC = (1ull << (r.x & 63)) - 1ull;
    t.lowM = (1ull << (r.y & 63)) - 1ull;
    return t;
}

// the pod's tile-local ranks (cpu, memory) in tile k
__device__ __forceinline__ uint2 tile_ranks(const PodThreshold& t, uint32_t k) {
    return make_uint2(__ldg(t.baseC + k) + __popcll(__ldg(t.membC + k) & t.lowC),
                      __ldg(t.baseM + k) + __popcll(__ldg(t.membM + k) & t.lowM));
}

// feasibility mask of tile k of a column-block index for one pod, from its tile-local ranks
template <int W>
__device__ __forceinline__ void ptile_mask(const uint8_t* __restrict__ blob, const RowsLayout& lay, uint2 rank,
                                           const unsigned long long (&sel)[W], uint32_t k, uint32_t (&m)[8]) {
    const uint8_t* cbp = blob + (size_t)(k / RW_TILES) * lay.cb_stride; // the tile's column block
    const uint32_t t32 = (k % RW_TILES) * 32;                          // the tile's bytes in every line of it
    const uint4* tc = reinterpret_cast<const uint4*>(cbp + (lay.off_tabC + rank.x * RW_LINE + t32));
    const uint4* tm = reinterpret_cast<const uint4*>(cbp + (lay.off_tabM + rank.y * RW_LINE + t32));
    const uint4 c0 = __ldg(tc), c1 = __ldg(tc + 1);
    const uint4 m0 = __ldg(tm), m1 = __ldg(tm + 1);
    m[0] = c0.x & m0.x; m[1] = c0.y & m0.y; m[2] = c0.z & m0.z; m[3] = c0.w & m0.w;
    m[4] = c1.x & m1.x; m[5] = c1.y & m1.y; m[6] = c1.z & m1.z; m[7] = c1.w & m1.w;
    const uint8_t* pairs = cbp + (lay.off_pairs + t32);
#pragma unroll
    for (int w = 0; w < W; w++) {
        unsigned long long bits = sel[w];
        while (bits) {
            const uint32_t bit = w * 64 + __ffsll((long long)bits) - 1;
            bits &= bits - 1;
            const uint4* col = reinterpret_cast<const uint4*>(pairs + (size_t)bit * RW_LINE);
            const uint4 q0 = __ldg(col);
            const uint4 q1 = __ldg(col + 1);
            m[0] &= q0.x; m[1] &= q0.y; m[2] &= q0.z; m[3] &= q0.w;
            m[4] &= q1.x; m[5] &= q1.y; m[6] &= q1.z; m[7] &= q1.w;
        }
    }
}

__device__ __forceinline__ int first_bit_256(const uint32_t (&m)[8]) {
    int first = -1;
#pragma unroll
    for (int j = 7; j >= 0; j--)
        if (m[j]) first = j * 32 + __ffs(m[j]) - 1;
    return first;
}

__device__ __forceinline__ void write_binding(const OutView& ov, const PodView& pv, const PeerOut& po, uint32_t p, int slot,
                                              const int32_t* __restrict__ ord_idx, const int64_t* __restrict__ ord_prio) {
    int32_t best = -1;
    int64_t score = 0;
    if (slot >= 0) {
        best = __ldg(ord_idx + slot);
        score = leftover_score(__ldg(ord_prio + slot), __ldg(pv.req_cpu + p), __ldg(pv.req_mem + p));
    }
    if (ov.node_idx) ov.node_idx[p] = best;
    if (ov.score) ov.score[p] = score;
    for (uint32_t k = 0; k < po.n; k++) { // fused all-gather: the same binding goes to every peer over NVLink
        po.idx[k][p] = best;
        po.score[k][p] = score;
    }
}

constexpr uint32_t FF_HEAD_TILES = 2;

template <int W>
__global__ void __launch_bounds__(256)
    k_first_fit_head(const uint8_t* __restrict__ blobP, TileBuckets bk, RowsLayout lay, const int32_t* __restrict__ ord_idx,
                     const int64_t* __restrict__ ord_prio, PodView pv, const uint2* __restrict__ rk, OutView ov,
                     uint32_t* __restrict__ tail_list, uint32_t* __restrict__ tail_count, PeerOut po, bool last_kernel,
                     const unsigned long long* __restrict__ live, uint32_t N) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p == 0) exchange_stamp(po, 0);
    if (threadIdx.x == 0) trace_start(TR_ARGMAX1_START);
    if (p < pv.P) {
        const uint2 r = __ldg(rk + p);
        const PodThreshold t = pod_threshold(bk, lay, r);
        unsigned long long sel[W];
        bool dead = r.x >= N || r.y >= N; // the request exceeds every node's free cpu / memory
#pragma unroll
        for (int w = 0; w < W; w++) {
            sel[w] = __ldg(pv.sel + (size_t)p * W + w);
            dead |= (sel[w] & ~__ldg(live + w)) != 0; // a required pair that no node carries
        }
        if (dead) { // infeasible everywhere: answered without scanning the 196 tiles in the tail kernel
            write_binding(ov, pv, po, p, -1, ord_idx, ord_prio);
        } else {
        uint32_t m0[8], m1[8];
        const uint32_t k1 = min(1u, lay.n_tiles - 1);
        // both tiles' bucket words first: their table rows are then requested together, one load round after them
        const uint2 r0 = tile_ranks(t, 0), r1 = tile_ranks(t, k1);
        ptile_mask<W>(blobP, lay, r0, sel, 0, m0);
        ptile_mask<W>(blobP, lay, r1, sel, k1, m1);
        int slot = first_bit_256(m0);
        if (slot < 0 && lay.n_tiles > 1) {
            const int s1 = first_bit_256(m1);
            if (s1 >= 0) slot = BP_TILE + s1;
        }
        if (slot >= 0 || lay.n_tiles <= FF_HEAD_TILES) write_binding(ov, pv, po, p, slot, ord_idx, ord_prio);
        else tail_list[atomicAdd(tail_count, 1u)] = p; // order of the list does not affect any result
        }
    }
    if (c_trace) {
        __syncthreads();
        if (threadIdx.x == 0) trace_end(TR_ARGMAX1_END);
    }
    if (last_kernel) exchange_signal(po); // no tail kernel follows: this rank's bindings are complete
}

template <int W>
__global__ void __launch_bounds__(256)
    k_first_fit_tail(const uint8_t* __restrict__ blobP, TileBuckets bk, RowsLayout lay, const int32_t* __restrict__ ord_idx,
                     const int64_t* __restrict__ ord_prio, PodView pv, const uint2* __restrict__ rk, OutView ov,
                     const uint32_t* __restrict__ tail_list, const uint32_t* __restrict__ tail_count, PeerOut po) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    const uint32_t n = *tail_count;
    if (blockIdx.x == 0 && threadIdx.x == 0) exchange_stamp(po, 4);
    if (threadIdx.x == 0) trace_start(TR_ARGMAX2_START);
    for (uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
        const uint32_t p = tail_list[i];
        const PodThreshold t = pod_threshold(bk, lay, __ldg(rk + p));
        unsigned long long sel[W];
#pragma unroll
        for (int w = 0; w < W; w++) sel[w] = __ldg(pv.sel + (size_t)p * W + w);
        int slot = -1;
        for (uint32_t k0 = FF_HEAD_TILES; k0 < lay.n_tiles; k0 += 32) {
            const uint32_t k = k0 + lane;
            int s = -1;
            if (k < lay.n_tiles) {
                uint32_t m[8];
                ptile_mask<W>(blobP, lay, tile_ranks(t, k), sel, k, m);
                s = first_bit_256(m);
            }
            const uint32_t b = __ballot_sync(0xffffffffu, s >= 0);
            if (b) { // lowest tile index = highest priority
                const int src = __ffs(b) - 1;
                slot = (int)((k0 + src) * BP_TILE) + __shfl_sync(0xffffffffu, s, src);
                break;
            }
        }
        if (lane == 0) write_binding(ov, pv, po, p, slot, ord_idx, ord_prio);
    }
    if (c_trace) {
        __syncthreads();
        if (threadIdx.x == 0) trace_end(TR_ARGMAX2_END);
    }
    exchange_signal(po); // the head kernel's stores completed before this kernel started
}

// ---- argmax of KS_SCORE_LEAST_ALLOCATED (not separable): bound-ordered scan with early exit ----
// Nodes are visited in descending order of least_alloc_bound (ties by node index), 256 at a time through the same
// table machinery (blobL); every feasible node of a tile is scored exactly; the scan stops as soon as the best exact
// score beats the bound of everything that follows.  One warp per pod: all lanes derive the tile's feasibility mask,
// lane l scores the set bits of word l&7 whose position is congruent to l>>3 mod 4; shuffle argmax per tile.
// Pods with a negative request (allowed by the ABI, never produced by a Kubernetes object) void the bound: they scan
// every tile, which is still exact.
struct NodeEval { // one row per slot of the bound order
    int64_t fc, fm, ac, am;
    double inv_ac, inv_am; // 1/alloc: quotient estimate, corrected to the exact floor below
    int32_t idx;
    int32_t pad;
};

// Single-precision view of the same row: in the common case it gives k_least_alloc the EXACT integer score of a cell
// without the 64-byte row and the two 64-bit divisions.  x = (float)free_cpu and y = (float)alloc_cpu when they are
// exactly representable (|free_cpu| < 2^24, 0 < alloc_cpu < 2^24; y = +inf for alloc_cpu <= 0, where the cpu term is 0
// by definition; NaN otherwise): for a request that is exact too, t = (x - r) * 100 is exact while t < 2^24, and the
// floor of the correctly rounded quotient t / y of two such integers IS floor((free_cpu - r) * 100 / alloc_cpu) (a
// quotient that is not an integer is at least 1 / y away from one, more than the rounding error t / y * 2^-24 for
// t < 2^24).  Memory is in bytes and does not fit: z = free_mem * 100 / alloc_mem and w = 100 / alloc_mem (both 0 for
// alloc_mem <= 0) give the real-valued quotient z - r * w with a relative error of a few 2^-24; its floor is known
// whenever no integer lies within the error bound (the kernel uses 2e-6 * (|z| + |r * w|) + 1e-3, > 8 x the worst case).
// k_build_eval writes the rows of one bound order, and this view too unless hint is null (only k_least_alloc reads it).
__global__ void __launch_bounds__(256)
    k_build_eval(NodeTable nt, const int32_t* __restrict__ ordL_idx, uint32_t Nord, NodeEval* __restrict__ ev,
                 float4* __restrict__ hint) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= Nord) return;
    const int32_t n = ordL_idx[s];
    NodeEval e;
    e.idx = n;
    e.pad = 0;
    if (n >= 0) {
        e.fc = nt.free_cpu[n];
        e.fm = nt.free_mem[n];
        e.ac = nt.alloc_cpu[n];
        e.am = nt.alloc_mem[n];
    } else {
        e.fc = e.fm = INT64_MIN;
        e.ac = e.am = 0;
    }
    e.inv_ac = e.ac > 0 ? 1.0 / (double)e.ac : 0.0;
    e.inv_am = e.am > 0 ? 1.0 / (double)e.am : 0.0;
    ev[s] = e;
    if (!hint) return;
    const float qnan = __int_as_float(0x7fc00000);
    const bool fc_exact = e.fc > -(1ll << 24) && e.fc < (1ll << 24);
    const double Sm = e.am > 0 ? (double)e.fm * 100.0 * e.inv_am : 0.0;
    hint[s] = make_float4(fc_exact ? (float)e.fc : qnan, e.ac <= 0 ? INFINITY : (e.ac < (1ll << 24) ? (float)e.ac : qnan), (float)Sm,
                          (float)(100.0 * e.inv_am));
}

// floor(x / d) for x >= 0, d > 0 (both < 2^63): double estimate, then exact correction in integers
__device__ __forceinline__ int64_t div_floor_pos(int64_t x, int64_t d, double inv_d) {
    int64_t q = (int64_t)((double)x * inv_d);
    int64_t r = x - q * d;
    while (r < 0) {
        q--;
        r += d;
    }
    while (r >= d) {
        q++;
        r -= d;
    }
    return q;
}

// exactly the expression of k_select_direct / the oracle (truncating division; x may be negative only when the
// request is negative, where the generic operator is used)
__device__ __forceinline__ int64_t least_alloc_score(const NodeEval& e, int64_t rc, int64_t rm) {
    int64_t pc = 0, pm = 0;
    if (e.ac > 0) {
        const int64_t x = (e.fc - rc) * 100;
        pc = x >= 0 ? div_floor_pos(x, e.ac, e.inv_ac) : x / e.ac;
    }
    if (e.am > 0) {
        const int64_t x = (e.fm - rm) * 100;
        pm = x >= 0 ? div_floor_pos(x, e.am, e.inv_am) : x / e.am;
    }
    return (pc + pm) / 2;
}

constexpr uint32_t LA_MAX_WARPS = 8;     // 256-thread CTAs at most
constexpr uint32_t LA_FIRST_WINDOW = 8;  // tiles of the first window (then 32 per window)

template <int W>
__global__ void __launch_bounds__(256)
    k_least_alloc(const uint8_t* __restrict__ blobL, TileBuckets bk, RowsLayout lay, const NodeEval* __restrict__ ev,
                  const float4* __restrict__ hint, const int64_t* __restrict__ ordL_s0, const int32_t* __restrict__ ordL_idx, PodView pv,
                  const uint2* __restrict__ rk, OutView ov, PeerOut po, const unsigned long long* __restrict__ live, uint32_t N) {
    const longlong2 amax = *reinterpret_cast<const longlong2*>(live + KS_MAX_LABEL_WORDS); // max allocatable cpu / memory
    __shared__ uint4 s_mask[LA_MAX_WARPS][32][2]; // per warp: the feasibility masks of the current window of tiles
    __shared__ int64_t s_top[LA_MAX_WARPS][32];   //           and the score bound of the first slot of each of them
    const uint32_t lane = threadIdx.x & 31, wq = lane & 7, quarter = lane >> 3, wid = threadIdx.x >> 5;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    uint32_t ne = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) exchange_stamp(po, 0);
    if (threadIdx.x == 0) trace_start(TR_ARGMAX1_START);
    for (uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < pv.P; p += warps) {
        const uint2 r = __ldg(rk + p);
        const PodThreshold t = pod_threshold(bk, lay, r);
        unsigned long long sel[W];
        bool dead = r.x >= N || r.y >= N; // the request exceeds every node's free cpu / memory
#pragma unroll
        for (int w = 0; w < W; w++) {
            sel[w] = __ldg(pv.sel + (size_t)p * W + w);
            dead |= (sel[w] & ~__ldg(live + w)) != 0; // a required pair that no node carries
        }
        const int64_t rc = __ldg(pv.req_cpu + p), rm = __ldg(pv.req_mem + p);
        const float rcf = (float)rc, rmf = (float)rm;
        const bool rc_exact = rc > -(1ll << 24) && rc < (1ll << 24); // (float)rc is rc
        const bool bounded = rc >= 0 && rm >= 0; // else the bound does not hold: no early exit
        // per-pod slack: floor((f-r)*100/a) <= floor(f*100/a) - floor(r*100/a) and a <= a_max, so every feasible cell
        // scores <= bound(n) - D with D = (rc*100/ac_max + rm*100/am_max) / 2 (a_max = INT64_MAX, no slack, when some
        // node has a <= 0: its term is 0 in score and bound alike)
        const int64_t D = bounded ? ((amax.x > 0 ? (rc * 100) / amax.x : 0) + (amax.y > 0 ? (rm * 100) / amax.y : 0)) / 2 : 0;
        int64_t best = INT64_MIN;
        int32_t bidx = -1;
        // The scan runs in windows of tiles: 8 tiles first (93 % of the pods of BASELINE C3 are done within them), then 32 at a
        // time.  Phase A: lane j derives the feasibility mask of tile k0 + j - the lanes work on DIFFERENT tiles, so the two
        // dependent rounds of table loads of a whole window overlap - and parks it in shared memory with the tile's top bound.
        // Phase B: the tiles that have a feasible slot at all are scored one by one, in bound order, by the whole warp.  Tiles
        // without a feasible slot cost nothing beyond phase A (a pod that fits nowhere no longer pays a full iteration per tile),
        // and the early exit is only evaluated in front of a tile that could change the result: the bounds descend, so it fires
        // there whenever it would have fired in front of an empty tile before it.
        uint32_t k0 = 0, win = LA_FIRST_WINDOW;
        bool done = dead;
        while (!done && k0 < lay.n_tiles) {
            if (k0 > 0 && bounded && bidx >= 0 && best > __ldg(ordL_s0 + (size_t)k0 * BP_TILE) - D) break; // warp-uniform
            {
                uint32_t m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
                int64_t top = INT64_MIN;
                const uint32_t kt = k0 + lane;
                if (lane < win && kt < lay.n_tiles) {
                    ptile_mask<W>(blobL, lay, tile_ranks(t, kt), sel, kt, m);
                    top = __ldg(ordL_s0 + (size_t)kt * BP_TILE);
                }
                s_mask[wid][lane][0] = make_uint4(m[0], m[1], m[2], m[3]);
                s_mask[wid][lane][1] = make_uint4(m[4], m[5], m[6], m[7]);
                s_top[wid][lane] = top;
                ne = __ballot_sync(0xffffffffu, (m[0] | m[1] | m[2] | m[3] | m[4] | m[5] | m[6] | m[7]) != 0u);
            }
            __syncwarp();
            while (ne) {
                const uint32_t j = __ffs(ne) - 1;
                ne &= ne - 1;
                const uint32_t k = k0 + j;
                if (bounded && bidx >= 0 && best > s_top[wid][j] - D) { // warp-uniform: nothing from here on can win or tie
                    done = true;
                    break;
                }
                // this lane's share of the tile's feasible slots: word wq, bit positions congruent to `quarter` mod 4
                const uint32_t bits = reinterpret_cast<const uint32_t*>(&s_mask[wid][j][0])[wq] & (0x11111111u << quarter);
                // Scores in single precision (k_build_eval): per feasible slot of this lane an interval [lo, hi] of integers that
                // contains the exact score - lo == hi (the score is KNOWN) unless the memory quotient lies within its error bound of
                // an integer, and [-inf, +inf] when the numbers leave the range in which the float arithmetic below is exact.  The
                // tile's winner scores >= max(lo), so only slots with hi >= max(max(lo), best so far) can win or tie: they load the
                // 4-byte node index (score known) or the 64-byte evaluation row for the exact 64-bit arithmetic (score not known).
                float hi[8];
                uint32_t known = 0; // bit i: lo == hi for this lane's i-th slot
                float lmax = -INFINITY;
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t b = quarter + 4u * i;
                    const bool f = (bits >> b) & 1u;
                    const float4 h = f ? __ldg(hint + (size_t)k * BP_TILE + wq * 32 + b) : make_float4(0.f, 1.f, 0.f, 0.f);
                    const float x = (h.x - rcf) * 100.0f;           // exact while it is an integer below 2^24
                    const float pc = floorf(__fdiv_rn(x, h.y));     // = floor((free_cpu - rc) * 100 / alloc_cpu); 0 for y = +inf
                    const float tm = rmf * h.w, qm = h.z - tm;      // memory quotient, real-valued estimate
                    const float em = 2e-6f * (fabsf(h.z) + fabsf(tm)) + 1e-3f;
                    const float pm_lo = h.w == 0.f ? 0.f : floorf(qm - em), pm_hi = h.w == 0.f ? 0.f : floorf(qm + em);
                    // every float sum below must be exact: integers under 2^23
                    const bool ok = rc_exact && x >= 0.f && x < 16777216.f && pc < 4.0e6f && fabsf(qm) + em < 4.0e6f; // false for NaN
                    const float lo = floorf((pc + pm_lo) * 0.5f);
                    hi[i] = f ? (ok ? floorf((pc + pm_hi) * 0.5f) : INFINITY) : -INFINITY;
                    if (f && ok) {
                        lmax = fmaxf(lmax, lo);
                        known |= (lo == hi[i] ? 1u : 0u) << i;
                    }
                }
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, off));
                bool changed = false;
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t b = quarter + 4u * i;
                    if (!((bits >> b) & 1u)) continue;              // not feasible
                    if (hi[i] < lmax) continue;                     // cannot reach the tile's winner
                    if (bidx >= 0 && hi[i] < (float)best) continue; // cannot reach the best so far (merged or this lane's)
                    const size_t slot = (size_t)k * BP_TILE + wq * 32 + b;
                    int64_t sc;
                    int32_t ni;
                    if ((known >> i) & 1u) {
                        sc = (int64_t)hi[i];
                        ni = __ldg(ordL_idx + slot);
                    } else {
                        const NodeEval e = ev[slot];
                        sc = least_alloc_score(e, rc, rm);
                        ni = e.idx;
                    }
                    if (sc > best || (sc == best && ni < bidx)) {
                        best = sc;
                        bidx = ni;
                        changed = true;
                    }
                }
                // every lane starts a tile with the same (best, bidx); merge only when some lane improved on it
                if (__any_sync(0xffffffffu, changed)) {
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) { // every lane ends with the tile-merged best
                        const int64_t os = __shfl_xor_sync(0xffffffffu, best, off);
                        const int32_t oi = __shfl_xor_sync(0xffffffffu, bidx, off);
                        if (oi >= 0 && (bidx < 0 || os > best || (os == best && oi < bidx))) {
                            best = os;
                            bidx = oi;
                        }
                    }
                }
            }
            __syncwarp(); // the next window overwrites this warp's slice of s_mask / s_top
            k0 += win;
            win = 32;
        }
        if (lane == 0) {
            const int64_t score = bidx >= 0 ? best : 0;
            if (ov.node_idx) ov.node_idx[p] = bidx;
            if (ov.score) ov.score[p] = score;
            for (uint32_t q = 0; q < po.n; q++) {
                po.idx[q][p] = bidx;
                po.score[q][p] = score;
            }
        }
    }
    if (c_trace) {
        __syncthreads();
        if (threadIdx.x == 0) trace_end(TR_ARGMAX1_END);
    }
    exchange_signal(po);
}

// ---- argmax of KS_SCORE_MOST_ALLOCATED: k_least_alloc's bound-ordered scan over an order of its own ----
// b(n) = term(f_c, A_c, 0) + term(f_m, A_m, 0) in [0, 200] (most_alloc_term, ks_internal.cuh).  For q >= 0,
// clamp(x + q) <= clamp(x) + q and floor((y + q) * 100 / A) <= floor(y * 100 / A) + ceil(q * 100 / A), and a term is at
// most 100, so every feasible cell of a pod with requests q >= 0 scores <= floor((b(n) + D) / 2) with
// D = min(100, ceil(q_c * 100 / m_c)) + min(100, ceil(q_m * 100 / m_m)), m the smallest positive allocatable (a node with
// A <= 0 has a term of 0 in score and bound alike).  Nodes are visited in descending b(n), ties by node index; the scan
// stops once that bound of everything left is strictly below the best exact score.  A negative request voids the bound.
// Built only when a MOST_ALLOCATED call needs it: one CTA sorts the nodes stably on 200 - b(n) (one 8-bit radix pass of
// ks_sort.cuh), then k_build_tiles and k_build_eval fill the tile index and the evaluation rows in that order.
// bound_order is that CTA for any order: `key' is the node's 8-bit sort digit (ascending = bound descending) and `val'
// the bound stored for it.
template <class Key, class Val>
__device__ __forceinline__ void bound_order(const NodeTable& nt, uint32_t Nord, uint32_t* __restrict__ buf,
                                            int32_t* __restrict__ ord_idx, int64_t* __restrict__ ord_b,
                                            long long* __restrict__ amin, Key key, Val val) {
    __shared__ SortShared s;
    __shared__ long long s_min[2];
    const uint32_t N = nt.N;
    if (threadIdx.x == 0) s_min[0] = s_min[1] = LLONG_MAX;
    __syncthreads();
    long long mc = LLONG_MAX, mm = LLONG_MAX;
    for (uint32_t i = threadIdx.x; i < N; i += SORT_THREADS) {
        buf[i] = i;
        const long long ac = nt.alloc_cpu[i], am = nt.alloc_mem[i];
        if (ac > 0) mc = min(mc, ac);
        if (am > 0) mm = min(mm, am);
    }
    atomicMin(&s_min[0], mc);
    atomicMin(&s_min[1], mm);
    __syncthreads();
    if (threadIdx.x == 0) {
        amin[0] = s_min[0];
        amin[1] = s_min[1];
    }
    cta_radix_pass(buf, buf + N, N, key, s);
    for (uint32_t k = threadIdx.x; k < Nord; k += SORT_THREADS) {
        const int32_t n = k < N ? (int32_t)buf[N + k] : -1;
        ord_idx[k] = n;
        ord_b[k] = n >= 0 ? val((uint32_t)n) : -1; // padding: below every bound, never feasible
    }
}
__global__ void __launch_bounds__(SORT_THREADS)
    k_most_order(NodeTable nt, uint32_t Nord, uint32_t* __restrict__ buf, int32_t* __restrict__ ord_idx,
                 int64_t* __restrict__ ord_b, long long* __restrict__ amin) {
    auto b = [&](uint32_t n) {
        return most_alloc_term(nt.free_cpu[n], nt.alloc_cpu[n], 0) + most_alloc_term(nt.free_mem[n], nt.alloc_mem[n], 0);
    };
    bound_order(nt, Nord, buf, ord_idx, ord_b, amin, [&](uint32_t n) { return (uint32_t)(200 - b(n)); }, b);
}

// ---- argmax of KS_SCORE_LEAST_BALANCED: the same scan over an order of its own (DESIGN.md 5j has the proof) ----
// b(n) = least_alloc_bound(n) + bal(n), bal(n) an integer upper bound of the balanced term at q = 0:
//   P_r = most_alloc_term(f_r, A_r, 0) = floor(100 * x_r(0)), so |x_c(0) - x_m(0)| > (|P_c - P_m| - 1) / 100 and
//   bal(n) = 100 - floor(max(0, |P_c - P_m| - 1) / 2) >= 100 - 50 * |x_c(0) - x_m(0)|   (100 when some A_r <= 0).
// For q >= 0 each share rises by at most min(1, q_r / m_r) <= C / 100, C = max_r min(100, ceil(q_r * 100 / m_r)), so the
// gap falls by at most C / 100 and the real-valued balanced term by at most C / 2; the double evaluation of balanced_int
// lies within 2^-43 of the real value, so trunc() of it is <= bal(n) + E with E = ceil(C / 2).  LEAST_ALLOCATED's
// per-pod slack D (k_least_alloc) bounds the other term: every feasible cell scores <= b(n) - D + E.  b(n) lies in
// [0, 200] unless free exceeds the allocatable or is negative: such nodes sort first with the bound LB_UNBOUNDED (no
// early exit while one is left), or last with the bound 0 (they are infeasible for q >= 0); either way the stored bound
// is >= b(n) and descending, which is all the early exit needs.
constexpr int64_t LB_UNBOUNDED = 1ll << 62; // above every b(n) inside the limits of ksched.h, and below 2^63 - any D
__device__ __forceinline__ int64_t balanced_bound(int64_t fc, int64_t fm, int64_t ac, int64_t am) {
    if (ac <= 0 || am <= 0) return 100;
    const int64_t d = llabs(most_alloc_term(fc, ac, 0) - most_alloc_term(fm, am, 0));
    return 100 - (d > 0 ? (d - 1) / 2 : 0);
}
__device__ __forceinline__ int64_t least_balanced_bound(const NodeTable& nt, uint32_t n) {
    return least_alloc_bound(nt, n) + balanced_bound(nt.free_cpu[n], nt.free_mem[n], nt.alloc_cpu[n], nt.alloc_mem[n]);
}
__global__ void __launch_bounds__(SORT_THREADS)
    k_balanced_order(NodeTable nt, uint32_t Nord, uint32_t* __restrict__ buf, int32_t* __restrict__ ord_idx,
                     int64_t* __restrict__ ord_b, long long* __restrict__ amin) {
    bound_order(
        nt, Nord, buf, ord_idx, ord_b, amin,
        [&](uint32_t n) { // 0: above 200; 1..201: 200 down to 0
            const int64_t b = least_balanced_bound(nt, n);
            return b > 200 ? 0u : (uint32_t)(201 - (b > 0 ? b : 0));
        },
        [&](uint32_t n) {
            const int64_t b = least_balanced_bound(nt, n);
            return b > 200 ? LB_UNBOUNDED : (b > 0 ? b : 0);
        });
}

// min(100, ceil(q * 100 / m)) for q >= 0, m > 0 (m may be LLONG_MAX: no node has a positive allocatable)
__device__ __forceinline__ int64_t most_alloc_slack(int64_t q, long long m) {
    const int64_t x = q * 100;
    const int64_t c = (int64_t)(x / m) + (x % m != 0 ? 1 : 0);
    return c < 100 ? c : 100;
}

// The highest score a cell in a slot with bound `top' can have: MOST_ALLOCATED (b + D) / 2, LEAST_BALANCED b - D
template <bool MOST>
__device__ __forceinline__ int64_t limit(int64_t top, int64_t D) { return MOST ? (top + D) / 2 : top - D; }

// The walk of k_most_alloc and k_least_balanced: k_least_alloc's windows over an order of their own, exact scores
// (alloc_score), and the early exit of each policy in front of every tile with a feasible slot.
template <int W, int POLICY>
__device__ __forceinline__ void bound_walk(const uint8_t* __restrict__ blob, const TileBuckets& bk, const RowsLayout& lay,
                                           const NodeEval* __restrict__ ev, const int64_t* __restrict__ ord_b,
                                           const long long* __restrict__ amin, const PodView& pv,
                                           const uint2* __restrict__ rk, const OutView& ov, const PeerOut& po,
                                           const unsigned long long* __restrict__ live, uint32_t N) {
    static_assert(POLICY == KS_SCORE_MOST_ALLOCATED || POLICY == KS_SCORE_LEAST_BALANCED, "a bound-ordered policy");
    constexpr bool MOST = POLICY == KS_SCORE_MOST_ALLOCATED;
    __shared__ uint4 s_mask[LA_MAX_WARPS][32][2]; // per warp: the feasibility masks of the current window of tiles
    __shared__ int64_t s_top[LA_MAX_WARPS][32];   //           and the bound of the first slot of each of them
    const uint32_t lane = threadIdx.x & 31, wq = lane & 7, quarter = lane >> 3, wid = threadIdx.x >> 5;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    const long long mc = __ldg(amin), mm = __ldg(amin + 1);
    uint32_t ne = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) exchange_stamp(po, 0);
    if (threadIdx.x == 0) trace_start(TR_ARGMAX1_START);
    for (uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < pv.P; p += warps) {
        const uint2 r = __ldg(rk + p);
        const PodThreshold t = pod_threshold(bk, lay, r);
        unsigned long long sel[W];
        bool dead = r.x >= N || r.y >= N; // the request exceeds every node's free cpu / memory
#pragma unroll
        for (int w = 0; w < W; w++) {
            sel[w] = __ldg(pv.sel + (size_t)p * W + w);
            dead |= (sel[w] & ~__ldg(live + w)) != 0; // a required pair that no node carries
        }
        const int64_t rc = __ldg(pv.req_cpu + p), rm = __ldg(pv.req_mem + p);
        const bool bounded = rc >= 0 && rm >= 0; // else the bound does not hold: no early exit
        // MOST_ALLOCATED: every feasible cell scores <= (b + D) / 2.  LEAST_BALANCED: <= b - D, D = LEAST_ALLOCATED's slack
        // (k_least_alloc) minus E
        int64_t D = 0;
        if (MOST) {
            D = bounded ? most_alloc_slack(rc, mc) + most_alloc_slack(rm, mm) : 0;
        } else if (bounded) {
            const longlong2 amax = *reinterpret_cast<const longlong2*>(live + KS_MAX_LABEL_WORDS);
            const int64_t dl = ((amax.x > 0 ? (rc * 100) / amax.x : 0) + (amax.y > 0 ? (rm * 100) / amax.y : 0)) / 2;
            const int64_t sc = most_alloc_slack(rc, mc), sm = most_alloc_slack(rm, mm);
            D = dl - ((sc > sm ? sc : sm) + 1) / 2;
        }
        int64_t best = INT64_MIN;
        int32_t bidx = -1;
        // windows of tiles as in k_least_alloc: phase A derives a window's feasibility masks (lane j: tile k0 + j), phase
        // B scores the tiles with a feasible slot in bound order; the early exit is tested in front of each of them
        uint32_t k0 = 0, win = LA_FIRST_WINDOW;
        bool done = dead;
        while (!done && k0 < lay.n_tiles) {
            if (k0 > 0 && bounded && bidx >= 0 && best > limit<MOST>(__ldg(ord_b + (size_t)k0 * BP_TILE), D))
                break; // warp-uniform
            {
                uint32_t m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
                int64_t top = INT64_MIN;
                const uint32_t kt = k0 + lane;
                if (lane < win && kt < lay.n_tiles) {
                    ptile_mask<W>(blob, lay, tile_ranks(t, kt), sel, kt, m);
                    top = __ldg(ord_b + (size_t)kt * BP_TILE);
                }
                s_mask[wid][lane][0] = make_uint4(m[0], m[1], m[2], m[3]);
                s_mask[wid][lane][1] = make_uint4(m[4], m[5], m[6], m[7]);
                s_top[wid][lane] = top;
                ne = __ballot_sync(0xffffffffu, (m[0] | m[1] | m[2] | m[3] | m[4] | m[5] | m[6] | m[7]) != 0u);
            }
            __syncwarp();
            while (ne) {
                const uint32_t j = __ffs(ne) - 1;
                ne &= ne - 1;
                const uint32_t k = k0 + j;
                if (bounded && bidx >= 0 && best > limit<MOST>(s_top[wid][j], D)) { // warp-uniform: nothing left can win or tie
                    done = true;
                    break;
                }
                // this lane's share of the tile's feasible slots: word wq, bit positions congruent to `quarter` mod 4
                const uint32_t bits = reinterpret_cast<const uint32_t*>(&s_mask[wid][j][0])[wq] & (0x11111111u << quarter);
                bool changed = false;
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t b = quarter + 4u * i;
                    if (!((bits >> b) & 1u)) continue;
                    const NodeEval e = ev[(size_t)k * BP_TILE + wq * 32 + b];
                    const int64_t sc = alloc_score<POLICY>(e.fc, e.fm, e.ac, e.am, rc, rm);
                    if (sc > best || (sc == best && e.idx < bidx)) {
                        best = sc;
                        bidx = e.idx;
                        changed = true;
                    }
                }
                if (__any_sync(0xffffffffu, changed)) {
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) { // every lane ends with the tile-merged best
                        const int64_t os = __shfl_xor_sync(0xffffffffu, best, off);
                        const int32_t oi = __shfl_xor_sync(0xffffffffu, bidx, off);
                        if (oi >= 0 && (bidx < 0 || os > best || (os == best && oi < bidx))) {
                            best = os;
                            bidx = oi;
                        }
                    }
                }
            }
            __syncwarp(); // the next window overwrites this warp's slice of s_mask / s_top
            k0 += win;
            win = 32;
        }
        if (lane == 0) {
            const int64_t score = bidx >= 0 ? best : 0;
            if (ov.node_idx) ov.node_idx[p] = bidx;
            if (ov.score) ov.score[p] = score;
            for (uint32_t q = 0; q < po.n; q++) {
                po.idx[q][p] = bidx;
                po.score[q][p] = score;
            }
        }
    }
    if (c_trace) {
        __syncthreads();
        if (threadIdx.x == 0) trace_end(TR_ARGMAX1_END);
    }
    exchange_signal(po);
}

template <int W>
__global__ void __launch_bounds__(256)
    k_most_alloc(const uint8_t* __restrict__ blobM, TileBuckets bk, RowsLayout lay, const NodeEval* __restrict__ ev,
                 const int64_t* __restrict__ ordM_b, const long long* __restrict__ amin, PodView pv,
                 const uint2* __restrict__ rk, OutView ov, PeerOut po, const unsigned long long* __restrict__ live, uint32_t N) {
    bound_walk<W, KS_SCORE_MOST_ALLOCATED>(blobM, bk, lay, ev, ordM_b, amin, pv, rk, ov, po, live, N);
}
template <int W>
__global__ void __launch_bounds__(256)
    k_least_balanced(const uint8_t* __restrict__ blobB, TileBuckets bk, RowsLayout lay, const NodeEval* __restrict__ ev,
                     const int64_t* __restrict__ ordB_b, const long long* __restrict__ amin, PodView pv,
                     const uint2* __restrict__ rk, OutView ov, PeerOut po, const unsigned long long* __restrict__ live,
                     uint32_t N) {
    bound_walk<W, KS_SCORE_LEAST_BALANCED>(blobB, bk, lay, ev, ordB_b, amin, pv, rk, ov, po, live, N);
}

// ------------------------------------------------------------------------------------------------ host side
// The column-block format (ks_bitpar.h) of all three indexes: column blocks of RW_TILES tiles; the mask kernel stages the
// pair columns with the tables when everything fits in shared memory (W <= 4), else it reads them through L1/L2
static bool make_layout_rows(uint32_t N, uint32_t W, RowsLayout* lay) {
    const uint32_t n_tiles = (N + BP_TILE - 1) / BP_TILE;
    if (n_tiles == 0) return false;
    lay->n_tiles = n_tiles;
    lay->ncb = (n_tiles + RW_TILES - 1) / RW_TILES;
    lay->off_tabC = 0;
    lay->off_tabM = RW_TAB_BYTES;
    lay->off_pairs = 2 * RW_TAB_BYTES;
    const uint32_t pairs_bytes = 64u * W * RW_LINE;
    lay->cb_stride = 2 * RW_TAB_BYTES + pairs_bytes; // multiple of 256
    lay->pairs_smem = lay->cb_stride <= (uint32_t)BP_SMEM_MAX - 1024u ? 1u : 0u;
    lay->smem_bytes = lay->pairs_smem ? lay->cb_stride : 2 * RW_TAB_BYTES;
    lay->n_thr = N + 1;
    // rank tables: 2 x ncb x (N+1) x 16 B; beyond 4 GB (N >= 2^19) the per-cell kernel serves the snapshot.  The largest
    // index this admits (N = 2^19 - 1, W = 8) has 64 MB blobs and 320 MB of bucket arrays per order.
    return (uint64_t)lay->ncb * lay->n_thr * RW_TILES * 2ull * 2ull <= (4ull << 30);
}

// The bucket arrays of an ordered index in one block (TileBuckets): base [resource][bucket][tile] u16, then memb
// [resource][bucket][tile] u64, rows of n_tiles entries (no argmax kernel reads a padding tile).  Returns the block's
// size; given the block, also sets *bk to the arrays in it.
static size_t tile_buckets(void* block, uint32_t N, const RowsLayout& lay, TileBuckets* bk) {
    const size_t n = ((size_t)(N >> 6) + 1) * lay.n_tiles;
    BlockLayout L;
    const size_t o_base = L.take<uint16_t>(2 * n), o_memb = L.take<unsigned long long>(2 * n);
    if (block)
        for (int r = 0; r < 2; r++) {
            bk->base[r] = at<uint16_t>(block, o_base) + r * n;
            bk->memb[r] = at<unsigned long long>(block, o_memb) + r * n;
        }
    return L.size;
}

BitparIndex::~BitparIndex() {
    if (trace.p) {
        unsigned long long* none = nullptr;
        cudaMemcpyToSymbol(c_trace, &none, sizeof(none));
    }
}

cudaError_t bitpar_build(BitparIndex& ix, const NodeTable& nt, int64_t* prio, cudaStream_t st) {
    ix.valid = false;
    ix.ordL.valid = false;
    ix.ordM.valid = ix.ordB.valid = false; // these orders follow on the next call that needs them (bitpar_prepare_order)
    ix.N = nt.N;
    ix.W = nt.W;
    if (nt.N == 0) return cudaSuccess;
    const uint32_t Nord = ((nt.N + BP_TILE - 1) / BP_TILE) * BP_TILE;
    ix.Nord = Nord;
    cudaError_t e;
    for (DevBuf* b : {&ix.sortedC, &ix.sortedM, &ix.ord_prio, &ix.ordL.b})
        if ((e = b->ensure((size_t)Nord * sizeof(int64_t))) != cudaSuccess) return e;
    for (DevBuf* b : {&ix.gposC, &ix.gposM, &ix.ord_idx, &ix.ordL.idx})
        if ((e = b->ensure((size_t)Nord * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = ix.ordL.eval.ensure((size_t)Nord * sizeof(NodeEval))) != cudaSuccess) return e;
    if ((e = ix.hintL.ensure((size_t)Nord * sizeof(float4))) != cudaSuccess) return e;
    for (DevBuf* b : {&ix.splC, &ix.splM})
        if ((e = b->ensure(RANK_SPLITTERS * sizeof(int64_t))) != cudaSuccess) return e;
    // [order][node], strided by N
    if ((e = ix.rk_bkt.ensure((size_t)N_ORDERS * nt.N * sizeof(uint8_t))) != cudaSuccess) return e;
    for (DevBuf* b : {&ix.rk_loc, &ix.rk_perm})
        if ((e = b->ensure((size_t)N_ORDERS * nt.N * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = ix.rk_hist.ensure(N_ORDERS * RANK_BUCKETS * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = ix.rk_spl_v.ensure(N_ORDERS * RANK_BUCKETS * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = ix.rk_spl_i.ensure(N_ORDERS * RANK_BUCKETS * sizeof(uint32_t))) != cudaSuccess) return e;
    uint32_t stride = 1;
    while ((nt.N + stride - 1) / stride > (uint32_t)RANK_SPLITTERS) stride <<= 1;
    ix.spl_stride = stride;
    ix.n_spl = (nt.N + stride - 1) / stride;
    const size_t live_bytes = (KS_MAX_LABEL_WORDS + 2) * sizeof(unsigned long long); // + max allocatable cpu, memory
    if ((e = ix.live.ensure(live_bytes)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(ix.live.p, 0, live_bytes, st)) != cudaSuccess) return e;
    k_node_bound<<<(nt.N + 255) / 256, 256, 0, st>>>(nt, prio + nt.Npad, ix.live.as<unsigned long long>());
    g_launches++;
    k_node_splitters<<<N_ORDERS, RANK_SAMPLES, 0, st>>>(nt, prio, ix.rk_spl_v.as<int64_t>(), ix.rk_spl_i.as<uint32_t>(),
                                                        ix.rk_hist.as<uint32_t>());
    k_node_bucket<<<(nt.N + 255) / 256, 256, 0, st>>>(nt, prio, ix.rk_spl_v.as<int64_t>(), ix.rk_spl_i.as<uint32_t>(),
                                                      ix.rk_hist.as<uint32_t>(), ix.rk_bkt.as<uint8_t>(),
                                                      ix.rk_loc.as<uint32_t>());
    k_node_scatter<<<(nt.N + 255) / 256, 256, 0, st>>>(nt.N, ix.rk_hist.as<uint32_t>(), ix.rk_bkt.as<uint8_t>(),
                                                       ix.rk_loc.as<uint32_t>(), ix.rk_perm.as<uint32_t>());
    k_node_rank<<<(Nord + 255) / 256, 256, 0, st>>>(
        nt, prio, ix.rk_hist.as<uint32_t>(), ix.rk_bkt.as<uint8_t>(), ix.rk_perm.as<uint32_t>(), ix.sortedC.as<int64_t>(),
        ix.sortedM.as<int64_t>(), ix.gposC.as<uint32_t>(), ix.gposM.as<uint32_t>(), ix.ord_prio.as<int64_t>(),
        ix.ord_idx.as<int32_t>(), Nord, ix.splC.as<int64_t>(), ix.splM.as<int64_t>(), stride, ix.ordL.b.as<int64_t>(),
        ix.ordL.idx.as<int32_t>());
    g_launches += 4;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    RowsLayout lay{};
    if (!make_layout_rows(nt.N, nt.W, &lay)) return cudaSuccess; // direct path only
    for (DevBuf* b : {&ix.blobR, &ix.blobP, &ix.ordL.blob})
        if ((e = b->ensure((size_t)lay.ncb * lay.cb_stride)) != cudaSuccess) return e;
    const size_t bucket_bytes = tile_buckets(nullptr, nt.N, lay, nullptr);
    for (DevBuf* b : {&ix.bucketsP, &ix.ordL.buckets})
        if ((e = b->ensure(bucket_bytes)) != cudaSuccess) return e;
    const size_t need_rank = (size_t)lay.ncb * lay.n_thr * 2 * (RW_TILES / 2); // u32 tile pairs
    if ((e = ix.rank.ensure(need_rank * sizeof(uint32_t))) != cudaSuccess) return e;
    // one work cursor per column block (k_mask_rows)
    if ((e = ix.cursor.ensure((size_t)lay.ncb * RW_CURSOR_STRIDE * sizeof(uint32_t))) != cudaSuccess) return e;
    const size_t need_ts = 2ull * lay.ncb * RW_TILES * BP_TILE;
    if ((e = ix.tile_sorted.ensure(need_ts * sizeof(uint32_t))) != cudaSuccess) return e;
    const uint32_t tiles = lay.ncb * RW_TILES;
    k_build_tiles<<<tiles, 288, 0, st>>>(nt, ix.gposC.as<uint32_t>(), ix.gposM.as<uint32_t>(), nullptr, ix.blobR.as<uint8_t>(),
                                         lay, ix.tile_sorted.as<uint32_t>(), TileBuckets{});
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    k_build_ranks<<<dim3((lay.n_thr + 255) / 256, lay.ncb), 256, 0, st>>>(ix.tile_sorted.as<uint32_t>(), lay,
                                                                           ix.rank.as<uint32_t>());
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    TileBuckets bk;
    tile_buckets(ix.bucketsP.p, nt.N, lay, &bk);
    k_build_tiles<<<tiles, 288, 0, st>>>(nt, ix.gposC.as<uint32_t>(), ix.gposM.as<uint32_t>(), ix.ord_idx.as<int32_t>(),
                                         ix.blobP.as<uint8_t>(), lay, nullptr, bk);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // KS_SCORE_LEAST_ALLOCATED: the same index in descending order of the score bound + per-slot evaluation rows
    tile_buckets(ix.ordL.buckets.p, nt.N, lay, &bk);
    k_build_tiles<<<tiles, 288, 0, st>>>(nt, ix.gposC.as<uint32_t>(), ix.gposM.as<uint32_t>(), ix.ordL.idx.as<int32_t>(),
                                         ix.ordL.blob.as<uint8_t>(), lay, nullptr, bk);
    k_build_eval<<<(Nord + 255) / 256, 256, 0, st>>>(nt, ix.ordL.idx.as<int32_t>(), Nord, ix.ordL.eval.as<NodeEval>(),
                                                     ix.hintL.as<float4>());
    g_launches += 2;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ix.lay_r = lay;
    ix.ordL.valid = ix.valid = true;
    return cudaSuccess;
}

// The order of a bound-ordered policy: KS_SCORE_LEAST_ALLOCATED, KS_SCORE_MOST_ALLOCATED or KS_SCORE_LEAST_BALANCED
static BoundOrder& bound_order(BitparIndex& ix, int policy) {
    return policy == KS_SCORE_LEAST_ALLOCATED ? ix.ordL : policy == KS_SCORE_MOST_ALLOCATED ? ix.ordM : ix.ordB;
}

cudaError_t bitpar_prepare_order(BitparIndex& ix, const NodeTable& nt, int policy, cudaStream_t st) {
    if (policy != KS_SCORE_MOST_ALLOCATED && policy != KS_SCORE_LEAST_BALANCED) return cudaSuccess;
    if (!ix.valid) return cudaErrorNotSupported;
    BoundOrder& o = bound_order(ix, policy);
    if (o.valid) return cudaSuccess;
    cudaError_t e;
    const uint32_t Nord = ix.Nord;
    if ((e = o.b.ensure((size_t)Nord * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = o.idx.ensure((size_t)Nord * sizeof(int32_t))) != cudaSuccess) return e;
    if ((e = o.eval.ensure((size_t)Nord * sizeof(NodeEval))) != cudaSuccess) return e;
    if ((e = o.sort.ensure(2ull * nt.N * sizeof(uint32_t) + 2 * sizeof(long long))) != cudaSuccess) return e;
    if ((e = o.blob.ensure((size_t)ix.lay_r.ncb * ix.lay_r.cb_stride)) != cudaSuccess) return e;
    if ((e = o.buckets.ensure(tile_buckets(nullptr, nt.N, ix.lay_r, nullptr))) != cudaSuccess) return e;
    long long* amin = reinterpret_cast<long long*>(o.sort.as<uint32_t>() + 2ull * nt.N);
    if (policy == KS_SCORE_MOST_ALLOCATED)
        k_most_order<<<1, SORT_THREADS, 0, st>>>(nt, Nord, o.sort.as<uint32_t>(), o.idx.as<int32_t>(), o.b.as<int64_t>(), amin);
    else
        k_balanced_order<<<1, SORT_THREADS, 0, st>>>(nt, Nord, o.sort.as<uint32_t>(), o.idx.as<int32_t>(), o.b.as<int64_t>(),
                                                     amin);
    TileBuckets bk;
    tile_buckets(o.buckets.p, nt.N, ix.lay_r, &bk);
    k_build_tiles<<<ix.lay_r.ncb * RW_TILES, 288, 0, st>>>(nt, ix.gposC.as<uint32_t>(), ix.gposM.as<uint32_t>(),
                                                          o.idx.as<int32_t>(), o.blob.as<uint8_t>(), ix.lay_r, nullptr, bk);
    k_build_eval<<<(Nord + 255) / 256, 256, 0, st>>>(nt, o.idx.as<int32_t>(), Nord, o.eval.as<NodeEval>(), nullptr);
    g_launches += 3;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    o.valid = true;
    return cudaSuccess;
}

// k_mask_rows' pod groups per chunk: about 20 chunks per CTA and column block, so that the CTAs sharing a block finish
// it close together, within RW_CHUNK_MIN..RW_CHUNK_MAX
static uint32_t rows_chunk(uint32_t n_groups, uint32_t ncb, uint32_t grid) {
    const uint32_t ctas_per_cb = std::max(1u, grid / ncb);
    return std::min(RW_CHUNK_MAX, std::max(RW_CHUNK_MIN, n_groups / (ctas_per_cb * 20u)));
}

bool bitpar_profitable(const BitparIndex& ix, uint32_t P) {
    // below ~16M cells the per-call rank pass and blob staging outweigh the per-cell kernel;
    // the mask kernel indexes (pod, tile) items with 32 bits
    return ix.valid && (uint64_t)P * ix.N >= (1ull << 24) && (uint64_t)P * RW_TILES < (1ull << 31);
}

template <int W, int THREADS>
static cudaError_t set_smem_attr1() {
    cudaError_t e = cudaFuncSetAttribute(k_mask_rows<W, W <= 4, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, BP_SMEM_MAX - 1024);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_count_rows<W, W <= 4, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, BP_SMEM_MAX - 1024);
}
template <int W>
static cudaError_t set_smem_attr() {
    cudaError_t e;
    if ((e = set_smem_attr1<W, 896>()) != cudaSuccess) return e;
    return set_smem_attr1<W, 960>();
}

// everything that allocates or configures: must run before a (possibly stream-captured) bitpar_select
cudaError_t bitpar_prepare(BitparIndex& ix, uint32_t P) {
    cudaError_t e;
    if (!ix.valid) return cudaErrorNotSupported;
    if (ix.sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&ix.sms, cudaDevAttrMultiProcessorCount, dev);
        if ((e = cudaStreamCreateWithFlags(&ix.aux.h, cudaStreamNonBlocking)) != cudaSuccess) return e;
        if ((e = cudaEventCreateWithFlags(&ix.ev_fork.h, cudaEventDisableTiming)) != cudaSuccess) return e;
        if ((e = cudaEventCreateWithFlags(&ix.ev_join.h, cudaEventDisableTiming)) != cudaSuccess) return e;
        if ((e = set_smem_attr<1>()) != cudaSuccess) return e;
        if ((e = set_smem_attr<2>()) != cudaSuccess) return e;
        if ((e = set_smem_attr<4>()) != cudaSuccess) return e;
        if ((e = set_smem_attr<8>()) != cudaSuccess) return e;
        if ((e = cudaFuncSetAttribute(k_pod_ranks, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      RANK_SPLITTERS * 2 * (int)sizeof(int64_t))) != cudaSuccess)
            return e;
        const char* tr = getenv("KS_TRACE");
        if (tr && tr[0] == '1') { // one trace buffer per device: the most recently prepared index owns the stamps
            if ((e = ix.trace.ensure(BP_TRACE_WORDS * sizeof(unsigned long long))) != cudaSuccess) return e;
            if ((e = cudaMemset(ix.trace.p, 0, BP_TRACE_WORDS * sizeof(unsigned long long))) != cudaSuccess) return e;
            if ((e = cudaMemcpyToSymbol(c_trace, &ix.trace.p, sizeof(ix.trace.p))) != cudaSuccess) return e;
        }
    }
    if ((e = ix.pod_ranks.ensure((size_t)P * sizeof(uint2))) != cudaSuccess) return e;
    if ((e = ix.tail_list.ensure(((size_t)P + 1) * sizeof(uint32_t))) != cudaSuccess) return e;
    if ((e = ix.rec_s.ensure((((size_t)P + 7) & ~(size_t)7) * sizeof(uint4))) != cudaSuccess) return e;
    return cudaSuccess;
}

template <int W>
static cudaError_t select_w(BitparIndex& ix, SelectLaunch& L, cudaEvent_t before_mask, cudaEvent_t after_mask) {
    cudaError_t e;
    const uint32_t P = L.pv.P;
    if ((uint64_t)P * RW_TILES >= (1ull << 31)) return cudaErrorInvalidValue;
    if ((e = bitpar_prepare(ix, P)) != cudaSuccess) return e; // no-op when the caller prepared already
    const bool need_mask_pass = L.ov.mask || L.ov.cnt;
    const int sms = ix.sms;
    if (ix.trace.p)
        if ((e = cudaMemsetAsync(ix.trace.p, 0, BP_TRACE_WORDS * sizeof(unsigned long long), L.stream)) != cudaSuccess) return e;
    // one 1024-thread CTA per SM (splitters in dynamic shared memory); two pods per thread and pass once P > #SMs * 1024
    const uint32_t rank_grid = (uint32_t)std::min<uint64_t>((uint64_t)sms, ((uint64_t)P + RANK_THREADS - 1) / RANK_THREADS);
    const size_t rank_smem = (size_t)ix.n_spl * 2 * sizeof(int64_t);
    const bool want_bind = L.ov.node_idx || L.ov.score;
    const bool overlap_bind = before_mask == nullptr && after_mask == nullptr;
    // How the mask kernel (persistent, one CTA per SM, SM-bound: every SM it does not get costs it 1/#SMs) and the argmax
    // kernels (latency-bound) share the chip.  Inside a CUDA graph the mask
    // kernel gets the SMs first, and a 256-thread argmax CTA does not fit beside a mask CTA (registers), so by default the
    // argmax kernels run after it.
    //   * short mask pass (< 256 MB of mask): the mask kernel leaves one SM in six to the argmax kernels, which then
    //     run beside it from the start; what they (and the exchange behind them) would add at the end costs more than the SMs.
    //   * long mask pass with an exchange attached: 896-thread mask CTAs + 128-thread argmax CTAs, which do fit beside them:
    //     the bindings go out to the peers early and the fences / flag latency hide under the mask kernel (the mask
    //     kernel pays for the company roughly what the argmax kernels cost alone, so without an exchange this buys nothing).
    //   * long mask pass, no exchange: 960-thread mask CTAs (fastest), argmax kernels behind them.
    const uint64_t mask_bytes = (uint64_t)P * (L.ov.mask ? L.ov.mask_row_words * 4ull : (uint64_t)ix.lay_r.n_tiles * 32ull);
    // (timing mode keeps the same shapes; it only moves the argmax kernels behind the mask kernel)
    const bool short_pass = need_mask_pass && want_bind && mask_bytes < (256ull << 20) && sms >= 48;
    const bool beside = !short_pass && need_mask_pass && want_bind && L.po.n > 0;
    const int threads = beside ? 896 : 960;
    const uint32_t at = beside ? 128u : 256u; // threads per argmax CTA
    const uint32_t mask_sms = short_pass ? (uint32_t)(sms - sms / 6) : (uint32_t)sms;
    const uint32_t n_groups = (P + 7) / 8;
    const uint64_t F = (uint64_t)n_groups * ix.lay_r.ncb;
    const uint32_t warps = (uint32_t)threads / 32;
    const uint32_t mask_grid = (uint32_t)std::min<uint64_t>((uint64_t)mask_sms, (F + warps - 1) / warps);
    k_pod_ranks<<<rank_grid, RANK_THREADS, rank_smem, L.stream>>>(L.pv, ix.sortedC.as<int64_t>(), ix.sortedM.as<int64_t>(), ix.N,
                                                 ix.splC.as<int64_t>(), ix.splM.as<int64_t>(), ix.n_spl, ix.spl_stride,
                                                 ix.pod_ranks.as<uint2>(), (need_mask_pass && ix.lay_r.ncb > 1) ? L.ov.cnt : nullptr, ix.W,
                                                 need_mask_pass ? ix.rec_s.as<uint4>() : nullptr, ix.cursor.as<uint32_t>(),
                                                 need_mask_pass ? ix.lay_r.ncb : 0u);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // argmax scan (needs only the pod ranks) on an auxiliary stream, forked here.  In timing mode it is enqueued on the main
    // stream behind the mask kernel instead, so that the event pair around the mask kernel times that kernel alone.
    if (want_bind) {
        if ((e = cudaEventRecord(ix.ev_fork, L.stream)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(ix.aux, ix.ev_fork, 0)) != cudaSuccess) return e;
    }
    auto enqueue_bind = [&](cudaStream_t bs) -> cudaError_t {
        uint32_t* tail_list = ix.tail_list.as<uint32_t>();
        uint32_t* tail_count = tail_list + P; // the list holds at most P pods
        if ((e = cudaMemsetAsync(tail_count, 0, sizeof(uint32_t), bs)) != cudaSuccess) return e;
        TileBuckets bk;
        if (L.policy != KS_SCORE_LEFTOVER) {
            const BoundOrder& o = bound_order(ix, L.policy);
            if (!o.valid) return cudaErrorNotSupported; // bitpar_prepare_order runs first
            tile_buckets(o.buckets.p, ix.N, ix.lay_r, &bk);
            const uint32_t wpc = at / 32; // one warp per pod
            const uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)sms * (2048 / at), ((uint64_t)P + wpc - 1) / wpc);
            if (L.policy == KS_SCORE_LEAST_ALLOCATED) {
                k_least_alloc<W><<<grid, at, 0, bs>>>(o.blob.as<uint8_t>(), bk, ix.lay_r, o.eval.as<NodeEval>(),
                                                      ix.hintL.as<float4>(), o.b.as<int64_t>(), o.idx.as<int32_t>(), L.pv,
                                                      ix.pod_ranks.as<uint2>(), L.ov, L.po,
                                                      ix.live.as<unsigned long long>(), ix.N);
            } else {
                const long long* amin = reinterpret_cast<const long long*>(o.sort.as<uint32_t>() + 2ull * ix.N);
                if (L.policy == KS_SCORE_MOST_ALLOCATED)
                    k_most_alloc<W><<<grid, at, 0, bs>>>(o.blob.as<uint8_t>(), bk, ix.lay_r, o.eval.as<NodeEval>(),
                                                         o.b.as<int64_t>(), amin, L.pv, ix.pod_ranks.as<uint2>(), L.ov,
                                                         L.po, ix.live.as<unsigned long long>(), ix.N);
                else
                    k_least_balanced<W><<<grid, at, 0, bs>>>(o.blob.as<uint8_t>(), bk, ix.lay_r, o.eval.as<NodeEval>(),
                                                             o.b.as<int64_t>(), amin, L.pv, ix.pod_ranks.as<uint2>(),
                                                             L.ov, L.po, ix.live.as<unsigned long long>(), ix.N);
            }
            g_launches++;
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
        } else {
            tile_buckets(ix.bucketsP.p, ix.N, ix.lay_r, &bk);
            const bool has_tail = ix.lay_r.n_tiles > FF_HEAD_TILES;
            k_first_fit_head<W><<<(P + at - 1) / at, at, 0, bs>>>(ix.blobP.as<uint8_t>(), bk, ix.lay_r, ix.ord_idx.as<int32_t>(),
                                                                 ix.ord_prio.as<int64_t>(), L.pv, ix.pod_ranks.as<uint2>(), L.ov,
                                                                 tail_list, tail_count, L.po, !has_tail,
                                                                 ix.live.as<unsigned long long>(), ix.N);
            g_launches++;
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            if (has_tail) {
                k_first_fit_tail<W><<<sms * (512 / at), at, 0, bs>>>(ix.blobP.as<uint8_t>(), bk, ix.lay_r, ix.ord_idx.as<int32_t>(),
                                                                     ix.ord_prio.as<int64_t>(), L.pv, ix.pod_ranks.as<uint2>(),
                                                                     L.ov, tail_list, tail_count, L.po);
                g_launches++;
                if ((e = cudaGetLastError()) != cudaSuccess) return e;
            }
        }
        // bindings are final here: start their device-to-host copy now, under the mask kernel
        if (L.host_node_idx && L.ov.node_idx) {
            if ((e = cudaMemcpyAsync(L.host_node_idx, L.ov.node_idx, (size_t)P * 4, cudaMemcpyDeviceToHost, bs)) != cudaSuccess) return e;
            L.host_node_idx = nullptr;
        }
        if (L.host_score && L.ov.score) {
            if ((e = cudaMemcpyAsync(L.host_score, L.ov.score, (size_t)P * 8, cudaMemcpyDeviceToHost, bs)) != cudaSuccess) return e;
            L.host_score = nullptr;
        }
        if (L.ready_event) { // tell the caller that node_idx / score are final (the mask pass may still be running)
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            if ((e = cudaStreamIsCapturing(bs, &cs)) != cudaSuccess) return e;
            e = cudaEventRecordWithFlags(L.ready_event, bs,
                                         cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault);
            if (e != cudaSuccess) return e;
            L.ready_event = nullptr;
        }
        return cudaSuccess;
    };
    if (want_bind && overlap_bind)
        if ((e = enqueue_bind(ix.aux)) != cudaSuccess) return e;
    if (need_mask_pass) {
        if (before_mask)
            if ((e = cudaEventRecord(before_mask, L.stream)) != cudaSuccess) return e;
        RowsParams prm;
        prm.blob = ix.blobR.as<uint8_t>();
        prm.lay = ix.lay_r;
        prm.rank = ix.rank.as<uint32_t>();
        prm.rec_s = ix.rec_s.as<uint4>();
        prm.sel_s = reinterpret_cast<const unsigned long long*>(L.pv.sel); // pod order: the caller's selector words
        prm.n_groups = n_groups;
        prm.mask = L.ov.mask;
        prm.row_words = (uint32_t)L.ov.mask_row_words;
        prm.cnt = L.ov.cnt;
        prm.cursor = ix.cursor.as<uint32_t>();
        prm.chunk = rows_chunk(n_groups, ix.lay_r.ncb, mask_grid);
        void (*kern)(RowsParams) = threads == 896 ? k_mask_rows<W, W <= 4, 896> : k_mask_rows<W, W <= 4, 960>;
        size_t smem = ix.lay_r.smem_bytes + RW_RING * prm.chunk * 128u;
        if (prm.mask == nullptr) { // counts only
            kern = threads == 896 ? k_count_rows<W, W <= 4, 896> : k_count_rows<W, W <= 4, 960>;
            smem = ix.lay_r.smem_bytes;
        }
        kern<<<mask_grid, threads, smem, L.stream>>>(prm);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (after_mask)
            if ((e = cudaEventRecord(after_mask, L.stream)) != cudaSuccess) return e;
    } else if (before_mask) {
        if ((e = cudaEventRecord(before_mask, L.stream)) != cudaSuccess) return e;
    }
    if (want_bind && !overlap_bind) // timing mode: on the main stream, behind the mask kernel
        if ((e = enqueue_bind(L.stream)) != cudaSuccess) return e;
    if (want_bind) { // join the auxiliary stream (it holds the argmax kernels unless timing mode put them on the main one)
        if ((e = cudaEventRecord(ix.ev_join, ix.aux)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(L.stream, ix.ev_join, 0)) != cudaSuccess) return e;
    }
    if (after_mask && !need_mask_pass)
        if ((e = cudaEventRecord(after_mask, L.stream)) != cudaSuccess) return e;
    return cudaSuccess;
}

cudaError_t bitpar_read_trace(const BitparIndex& ix, unsigned long long out_ns[BP_TRACE_WORDS]) {
    if (!ix.trace.p) return cudaErrorNotSupported;
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return e;
    if ((e = cudaMemcpy(out_ns, ix.trace.p, BP_TRACE_WORDS * sizeof(unsigned long long), cudaMemcpyDeviceToHost)) != cudaSuccess) return e;
    if (out_ns[TR_MASK_FIRST_CTA_END_INV]) out_ns[TR_MASK_FIRST_CTA_END_INV] = ~out_ns[TR_MASK_FIRST_CTA_END_INV];
    return cudaSuccess;
}

cudaError_t bitpar_select(BitparIndex& ix, SelectLaunch& L, cudaEvent_t before_mask, cudaEvent_t after_mask) {
    if (!ix.valid) return cudaErrorNotSupported;
    return with_label_width(ix.W, [&](auto w) { return select_w<decltype(w)::value>(ix, L, before_mask, after_mask); });
}

} // namespace ks
