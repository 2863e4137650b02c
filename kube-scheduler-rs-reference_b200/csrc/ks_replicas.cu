// ks_replicas.cu — replica placement (ks_place_replicas, include/ksched.h; DESIGN.md 5h), sm_90a.
// Copy j of a spec on node n scores s_n(j), non-increasing in j, so placing the copies one at a time by argmax is taking
// the first R' of all (node, copy) pairs by (score descending, node, copy).  Instead of R' dependent rounds:
//   k_rep_scan    per (node chunk, spec): k_n = min(c_n, R), and per chunk the capacity, feasible count, sum of k_n and
//                 the score bounds;
//   k_rep_init    per spec: R' and the bracket [min s_n(k_n - 1), max s_n(0)] of the threshold S*, the largest S with
//                 G(S) = sum_n #{j < k_n : s_n(j) >= S} >= R' (the score of copy R' - 1);
//   k_rep_count / k_rep_narrow, REP_PASSES times: G at 32 probes of the bracket (one per lane), then the bracket shrinks
//                 to the gap between two probes.  A spec whose bracket has closed returns at once;
//   k_rep_tally / k_rep_settle: a_n = G_n(S* + 1) copies above S*, e_n = G_n(S*) - a_n at it; the R' - sum a_n tied
//                 copies go to the lowest nodes (chunk prefixes here, the prefix inside a chunk in k_rep_emit);
//   k_rep_emit    count_n, the row's node count and maximum and, with the copy list, every copy in node-then-copy order;
//   k_rep_order   one CTA per spec: the stable radix sort of ks_sort.cuh on top - score, which is placement order.
// Under MOST_ALLOCATED s_n(j) is non-decreasing in j instead, and placement fills whole nodes in order of s_n(0) descending,
// node ascending (include/ksched.h).  The same kernels compute that plan with G_n(S) = s_n(0) >= S ? k_n : 0: S* is the
// s_n(0) of the last node that takes copies, the nodes above it take all k_n, the tie split fills the nodes at S* in node
// order, and k_rep_order_most sorts on top - s_n(0) of each copy's node, which keeps a node's copies together.
// Under LEAST_BALANCED s_n(j) can rise or fall with j, and neither shortcut holds: after k_rep_scan and k_rep_init,
// k_rep_seq places the copies one at a time, one CTA per spec (specs strided over a grid sized to a scratch budget).
#include "ks_launch.h"
#include "ks_replicas.cuh"
#include "ks_sort.cuh"

namespace ks {

constexpr int REP_PROBES = 32; // thresholds per search pass, one per lane
// The score of a placed copy lies in [0, 2^61): free after the copy is >= 0 and free <= 2^36 m / 2^55 B, so LEFTOVER's
// score is at most 2^58 + 2^55, and LEAST_ALLOCATED's at most (100 * 2^36 + 100 * 2^55) / 2 < 2^61 (an allocatable of
// 1 m and 1 B).  A pass leaves a bracket below 1/32 of the one it started with, so 13 passes (32^13 = 2^65) close
// every bracket.
constexpr int REP_PASSES = 13;
constexpr int REP_SCORE_BITS = 61;
static_assert(5 * REP_PASSES >= REP_SCORE_BITS, "the passes must close a bracket of 2^61 scores");
static_assert(REP_THREADS == SORT_THREADS, "k_rep_order and k_rep_emit use ks_sort.cuh's 256-thread scan and sort");

struct RepSpec {
    int64_t lo, hi;           // bracket of S*: G(lo) >= need and S* <= hi; lo == hi = S* once closed
    int64_t top;              // highest s_n(0): a copy's sort key is top - score
    uint64_t need;            // R' = min(replicas, sum of k_n)
    uint64_t tied;            // R' - G(S* + 1): the copies at score S*, taken by the lowest nodes
    uint64_t cnt[REP_PROBES]; // G at the probes of the current pass
};
struct RepChunk {
    uint64_t cap, sumk;   // capacity (saturating) and sum of k_n over the chunk's nodes
    uint64_t a, e;        // sums of a_n and e_n
    uint64_t e_pre, c_pre; // exclusive prefixes over the spec's chunks: of e, and of the placed copies
    int64_t hi, lo;       // max s_n(0), min s_n(k_n - 1) over the chunk's nodes with k_n >= 1
    uint32_t feas, pad;
};

// k_rep_seq: a CTA keeps the current score of every node (int64, INT64_MIN once it holds no further copy) and its copies
// placed so far (uint32) in device scratch, and the maximum of every block of `block' nodes, with its node, in shared
// memory.  block = 1024 nodes up to REP_SEQ_BLOCKS * 1024 nodes, larger beyond.
constexpr uint32_t REP_SEQ_BLOCKS = 2048;
constexpr uint64_t REP_SEQ_BUDGET = 64ull << 20; // scratch of all k_rep_seq CTAs of a call (at least one CTA's)
constexpr uint32_t REP_SEQ_NODE_BYTES = 12;

void replica_seq_grid(uint32_t N, uint32_t T, int sms, uint32_t* ctas, uint32_t* block) {
    const uint64_t fit = std::max<uint64_t>(1, REP_SEQ_BUDGET / ((uint64_t)std::max(N, 1u) * REP_SEQ_NODE_BYTES));
    *ctas = (uint32_t)std::min<uint64_t>(std::min<uint64_t>(fit, std::max(T, 1u)), 2ull * (uint64_t)std::max(sms, 1));
    const uint32_t per = 1024u * REP_SEQ_BLOCKS;
    *block = 1024u * std::max(1u, (N + per - 1) / per);
}

size_t replica_spec_bytes(uint32_t T) { return (size_t)T * sizeof(RepSpec); }
size_t replica_chunk_bytes(uint32_t T, uint32_t n_chunks) { return (size_t)T * n_chunks * sizeof(RepChunk); }

// Node chunks of REP_THREADS-node tiles: about 4 CTAs per SM over all specs, at least one tile per chunk.
void replica_chunks(uint32_t N, uint32_t T, int sms, uint32_t* n_chunks, uint32_t* chunk_len) {
    const uint32_t tiles = std::max(1u, (N + REP_THREADS - 1) / REP_THREADS);
    const uint32_t want = std::min(tiles, std::max(1u, (4u * (uint32_t)std::max(sms, 1) + T - 1) / std::max(T, 1u)));
    const uint32_t per = (tiles + want - 1) / want;
    *chunk_len = per * REP_THREADS;
    *n_chunks = (tiles + per - 1) / per;
}

// G_n(S) = #{j < k : s_n(j) >= S}.  LEFTOVER: s_n(j) = key_n - (j + 1) * d, a closed form.  LEAST_ALLOCATED: a binary
// search over j, after the bounds s0 = s_n(0) and sl = s_n(k - 1).  MOST_ALLOCATED: not that count but the copies a
// node filled in s_n(0) order holds, s0 >= S ? k : 0.
template <int POL>
__device__ __forceinline__ uint32_t rep_at(const RepNode& v, int64_t rc, int64_t rm, int64_t s0, int64_t sl, int64_t S) {
    if (v.k == 0) return 0;
    if (POL == KS_SCORE_LEFTOVER) {
        const int64_t x = leftover_key(v.fc, v.fm) - S, d = leftover_key(rc, rm);
        if (x < d) return 0; // even copy 0 (key_n - d) is below S
        return d == 0 ? v.k : (uint32_t)min((uint64_t)v.k, (uint64_t)x / (uint64_t)d);
    }
    if (S > s0) return 0;
    if (POL == KS_SCORE_MOST_ALLOCATED) return v.k;
    if (S <= sl) return v.k;
    uint32_t a = 1, b = v.k - 1; // s(a - 1) >= S > s(b)
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (rep_score<POL>(v, rc, rm, mid) >= S) a = mid + 1;
        else b = mid;
    }
    return a;
}

__device__ __forceinline__ uint64_t sat_add(uint64_t a, uint64_t b) { return a + b < a ? ~0ull : a + b; }

// What every (chunk, spec) kernel reads of its spec
template <int W>
struct RepCtx {
    int64_t rc, rm;
    uint64_t sel[W];
    uint32_t R, n0, n1;
    __device__ __forceinline__ RepCtx(const NodeTable& nt, const ReplicaArgs& a, uint32_t t, uint32_t c) {
        rc = a.req_cpu[t];
        rm = a.req_mem[t];
#pragma unroll
        for (int w = 0; w < W; w++) sel[w] = a.sel[(uint64_t)t * W + w];
        R = a.replicas[t];
        n0 = min(nt.N, c * a.chunk_len);
        n1 = min(nt.N, n0 + a.chunk_len);
    }
};

template <int W, int POL>
__global__ void __launch_bounds__(REP_THREADS) k_rep_scan(NodeTable nt, ReplicaArgs a) {
    __shared__ uint64_t red[REP_WARPS];
    const uint32_t t = blockIdx.y, c = blockIdx.x;
    const RepCtx<W> x(nt, a, t, c);
    uint64_t cap = 0, sumk = 0, feas = 0;
    int64_t hi = INT64_MIN, lo = INT64_MAX;
    for (uint32_t n = x.n0 + threadIdx.x; n < x.n1; n += REP_THREADS) {
        RepNode v;
        uint64_t cn;
        rep_node<W, POL>(nt, n, x.rc, x.rm, x.sel, x.R, v, cn);
        if (cn == 0) continue;
        feas++;
        cap = sat_add(cap, cn);
        sumk += v.k;
        if (v.k && POL != KS_SCORE_LEAST_BALANCED) { // k_rep_seq needs no bracket
            hi = max(hi, rep_score<POL>(v, x.rc, x.rm, 0));
            lo = min(lo, rep_score<POL>(v, x.rc, x.rm, POL == KS_SCORE_MOST_ALLOCATED ? 0 : v.k - 1));
        }
    }
    cap = rep_reduce(cap, sat_add, red);
    sumk = rep_reduce(sumk, [](uint64_t p, uint64_t q) { return p + q; }, red);
    feas = rep_reduce(feas, [](uint64_t p, uint64_t q) { return p + q; }, red);
    hi = rep_reduce(hi, [](int64_t p, int64_t q) { return max(p, q); }, reinterpret_cast<int64_t*>(red));
    lo = rep_reduce(lo, [](int64_t p, int64_t q) { return min(p, q); }, reinterpret_cast<int64_t*>(red));
    if (threadIdx.x == 0) {
        RepChunk& ch = a.chunk[(uint64_t)t * a.n_chunks + c];
        ch.cap = cap;
        ch.sumk = sumk;
        ch.feas = (uint32_t)feas;
        ch.hi = hi;
        ch.lo = lo;
    }
}

// One thread per spec: the row's capacity, feasible count and placed, and the search bracket.
__global__ void k_rep_init(ReplicaArgs a) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.T) return;
    const RepChunk* ch = a.chunk + (uint64_t)t * a.n_chunks;
    uint64_t cap = 0, sumk = 0;
    uint32_t feas = 0;
    int64_t hi = INT64_MIN, lo = INT64_MAX;
    for (uint32_t c = 0; c < a.n_chunks; c++) {
        cap = sat_add(cap, ch[c].cap);
        sumk += ch[c].sumk;
        feas += ch[c].feas;
        hi = max(hi, ch[c].hi);
        lo = min(lo, ch[c].lo);
    }
    const uint64_t need = min(sumk, (uint64_t)a.replicas[t]);
    RepSpec& sp = a.spec[t];
    sp.lo = need ? lo : 0;
    sp.hi = need ? hi : 0;
    sp.top = sp.hi;
    sp.need = need;
    sp.tied = 0;
    for (int i = 0; i < REP_PROBES; i++) sp.cnt[i] = 0;
    ks_replica_plan r;
    r.capacity = cap;
    r.placed = (uint32_t)need;
    r.nodes = 0;
    r.feasible_cnt = feas;
    r.max_per_node = 0;
    r.last_score = 0;
    a.rows[t] = r;
}

// Probe i of the bracket [lo, hi], lo < hi: lo + ceil((hi - lo) * (i + 1) / 32), so probe 31 is hi.  The product
// (up to 2^61 * 32) is taken in 128 bits.
__device__ __forceinline__ int64_t rep_probe(int64_t lo, int64_t hi, uint32_t i) {
    const unsigned __int128 x = (unsigned __int128)(uint64_t)(hi - lo) * (i + 1) + (REP_PROBES - 1);
    return lo + (int64_t)(uint64_t)(x / REP_PROBES);
}

// G at the 32 probes over one chunk: the warp walks its nodes, each lane evaluates its own probe.
template <int W, int POL>
__global__ void __launch_bounds__(REP_THREADS) k_rep_count(NodeTable nt, ReplicaArgs a) {
    __shared__ uint64_t part[REP_WARPS][32];
    const uint32_t t = blockIdx.y, c = blockIdx.x;
    RepSpec& sp = a.spec[t];
    const int64_t L = sp.lo, H = sp.hi;
    if (L == H) return; // closed, or nothing to place
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t S = rep_probe(L, H, lane);
    const RepCtx<W> x(nt, a, t, c);
    uint64_t cnt = 0;
    for (uint32_t b = x.n0 + warp * 32; b < x.n1; b += REP_THREADS) { // warp-uniform
        const uint32_t n = b + lane;
        RepNode v{0, 0, 0, 0, 0};
        int64_t s0 = 0, sl = 0;
        if (n < x.n1) {
            uint64_t cn;
            rep_node<W, POL>(nt, n, x.rc, x.rm, x.sel, x.R, v, cn);
            if (POL != KS_SCORE_LEFTOVER && v.k) {
                s0 = rep_score<POL>(v, x.rc, x.rm, 0);
                sl = POL == KS_SCORE_MOST_ALLOCATED ? s0 : rep_score<POL>(v, x.rc, x.rm, v.k - 1); // MOST: rep_at reads s0 only
            }
        }
        for (uint32_t live = __ballot_sync(0xffffffffu, v.k != 0); live; live &= live - 1) {
            const int src = __ffs(live) - 1;
            RepNode u;
            u.fc = __shfl_sync(0xffffffffu, v.fc, src);
            u.fm = __shfl_sync(0xffffffffu, v.fm, src);
            u.ac = __shfl_sync(0xffffffffu, v.ac, src);
            u.am = __shfl_sync(0xffffffffu, v.am, src);
            u.k = __shfl_sync(0xffffffffu, v.k, src);
            const int64_t u0 = __shfl_sync(0xffffffffu, s0, src), ul = __shfl_sync(0xffffffffu, sl, src);
            cnt += rep_at<POL>(u, x.rc, x.rm, u0, ul, S);
        }
    }
    part[warp][lane] = cnt;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint64_t sum = 0;
#pragma unroll
        for (int w = 0; w < REP_WARPS; w++) sum += part[w][threadIdx.x];
        if (sum) atomicAdd(reinterpret_cast<unsigned long long*>(&sp.cnt[threadIdx.x]), (unsigned long long)sum);
    }
}

// One thread per spec: keep the gap between the highest probe with G >= need and the probe after it.
__global__ void k_rep_narrow(ReplicaArgs a) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.T) return;
    RepSpec& sp = a.spec[t];
    const int64_t L = sp.lo, H = sp.hi;
    if (L == H) return;
    int best = -1; // G is non-increasing in the probe: the probes with G >= need are a prefix
    for (int i = 0; i < REP_PROBES; i++) {
        if (sp.cnt[i] >= sp.need) best = i;
        sp.cnt[i] = 0;
    }
    if (best < 0) {
        sp.hi = rep_probe(L, H, 0) - 1;
    } else {
        sp.lo = rep_probe(L, H, best);
        if (best + 1 < REP_PROBES) sp.hi = rep_probe(L, H, best + 1) - 1;
    }
}

// Per chunk: the copies above S* and the tied copies at S*.
template <int W, int POL>
__global__ void __launch_bounds__(REP_THREADS) k_rep_tally(NodeTable nt, ReplicaArgs a) {
    __shared__ uint64_t red[REP_WARPS];
    const uint32_t t = blockIdx.y, c = blockIdx.x;
    const RepSpec& sp = a.spec[t];
    uint64_t sa = 0, se = 0;
    if (sp.need) {
        const int64_t S = sp.lo;
        const RepCtx<W> x(nt, a, t, c);
        for (uint32_t n = x.n0 + threadIdx.x; n < x.n1; n += REP_THREADS) {
            RepNode v;
            uint64_t cn;
            rep_node<W, POL>(nt, n, x.rc, x.rm, x.sel, x.R, v, cn);
            if (!v.k) continue;
            const int64_t s0 = rep_score<POL>(v, x.rc, x.rm, 0);
            const int64_t sl = POL == KS_SCORE_MOST_ALLOCATED ? s0 : rep_score<POL>(v, x.rc, x.rm, v.k - 1);
            const uint32_t above = rep_at<POL>(v, x.rc, x.rm, s0, sl, S + 1);
            sa += above;
            se += rep_at<POL>(v, x.rc, x.rm, s0, sl, S) - above;
        }
    }
    sa = rep_reduce(sa, [](uint64_t p, uint64_t q) { return p + q; }, red);
    se = rep_reduce(se, [](uint64_t p, uint64_t q) { return p + q; }, red);
    if (threadIdx.x == 0) {
        RepChunk& ch = a.chunk[(uint64_t)t * a.n_chunks + c];
        ch.a = sa;
        ch.e = se;
    }
}

// One thread per spec: the tied count, the chunk prefixes and the row's last score.
__global__ void k_rep_settle(ReplicaArgs a) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.T) return;
    RepSpec& sp = a.spec[t];
    if (!sp.need) return;
    RepChunk* ch = a.chunk + (uint64_t)t * a.n_chunks;
    uint64_t above = 0;
    for (uint32_t c = 0; c < a.n_chunks; c++) above += ch[c].a;
    // G(S* + 1) < need by the choice of S*; the clamp keeps the tie split inside the spec's slot regardless
    const uint64_t K = sp.need > above ? sp.need - above : 0;
    uint64_t e_run = 0, c_run = 0;
    for (uint32_t c = 0; c < a.n_chunks; c++) {
        ch[c].e_pre = e_run;
        ch[c].c_pre = c_run;
        c_run += ch[c].a + (K > e_run ? min(ch[c].e, K - e_run) : 0);
        e_run += ch[c].e;
    }
    sp.tied = K;
    a.rows[t].last_score = sp.lo;
}

// count_n = a_n + min(e_n, max(0, K - prefix_n)) with prefix_n the exclusive prefix of e over the nodes; the row's node
// count and maximum; with the copy list, copy j of node n at its node-then-copy position.
template <int W, int POL>
__global__ void __launch_bounds__(REP_THREADS) k_rep_emit(NodeTable nt, ReplicaArgs a) {
    __shared__ uint32_t wsum[SORT_WARPS];
    __shared__ uint32_t red[REP_WARPS];
    const uint32_t t = blockIdx.y, c = blockIdx.x;
    const RepSpec& sp = a.spec[t];
    if (!sp.need) return;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t S = sp.lo;
    const uint64_t K = sp.tied, off = a.offset[t];
    const RepChunk& ch = a.chunk[(uint64_t)t * a.n_chunks + c];
    uint64_t e_run = ch.e_pre, c_run = ch.c_pre;
    const RepCtx<W> x(nt, a, t, c);
    uint32_t nodes = 0, most = 0;
    for (uint32_t b = x.n0; b < x.n1; b += REP_THREADS) { // block-uniform
        const uint32_t n = b + threadIdx.x;
        RepNode v{0, 0, 0, 0, 0};
        uint32_t above = 0, e = 0;
        if (n < x.n1) {
            uint64_t cn;
            rep_node<W, POL>(nt, n, x.rc, x.rm, x.sel, x.R, v, cn);
            if (v.k) {
                const int64_t s0 = rep_score<POL>(v, x.rc, x.rm, 0);
            const int64_t sl = POL == KS_SCORE_MOST_ALLOCATED ? s0 : rep_score<POL>(v, x.rc, x.rm, v.k - 1);
                above = rep_at<POL>(v, x.rc, x.rm, s0, sl, S + 1);
                e = rep_at<POL>(v, x.rc, x.rm, s0, sl, S) - above;
            }
        }
        uint32_t e_tot, c_tot;
        const uint64_t pre = e_run + cta_block_scan(e, wsum, e_tot);
        const uint32_t cnt = above + (K > pre ? (uint32_t)min((uint64_t)e, K - pre) : 0u);
        // MOST_ALLOCATED: the last copy placed is the last one of the node at S* whose tied copies reach K
        if (POL == KS_SCORE_MOST_ALLOCATED && e && pre < K && K <= pre + e)
            a.rows[t].last_score = rep_score<POL>(v, x.rc, x.rm, cnt - 1);
        const uint64_t base = off + c_run + cta_block_scan(cnt, wsum, c_tot);
        e_run += e_tot;
        c_run += c_tot;
        nodes += cnt != 0;
        most = max(most, cnt);
        if (!a.out_node) continue;
        for (uint32_t live = __ballot_sync(0xffffffffu, cnt != 0); live; live &= live - 1) {
            const int src = __ffs(live) - 1;
            RepNode u;
            u.fc = __shfl_sync(0xffffffffu, v.fc, src);
            u.fm = __shfl_sync(0xffffffffu, v.fm, src);
            u.ac = __shfl_sync(0xffffffffu, v.ac, src);
            u.am = __shfl_sync(0xffffffffu, v.am, src);
            const uint64_t bs = __shfl_sync(0xffffffffu, base, src);
            const uint64_t end = off + sp.need; // never past the spec's placed copies
            const uint32_t m = bs < end ? (uint32_t)min((uint64_t)__shfl_sync(0xffffffffu, cnt, src), end - bs) : 0u;
            const int32_t node = (int32_t)(b + warp * 32 + src);
            for (uint32_t j = lane; j < m; j += 32) {
                a.copy_node[bs + j] = node;
                a.copy_score[bs + j] = rep_score<POL>(u, x.rc, x.rm, j);
            }
        }
    }
    nodes = rep_reduce(nodes, [](uint32_t p, uint32_t q) { return p + q; }, red);
    most = rep_reduce(most, [](uint32_t p, uint32_t q) { return max(p, q); }, red);
    if (threadIdx.x == 0) {
        if (nodes) atomicAdd(&a.rows[t].nodes, nodes);
        if (most) atomicMax(&a.rows[t].max_per_node, most);
    }
}

// One CTA per spec: the copies, laid out node then copy, sorted stably by key(top, scores, t, nodes, i) (ascending; top - the
// copy's score, or top - s_n(0) of its node) are in placement order; only the digits of top - S* are sorted.
template <class Key>
__device__ __forceinline__ void rep_order(const ReplicaArgs& a, Key key) {
    __shared__ SortShared s;
    for (uint32_t t = blockIdx.x; t < a.T; t += gridDim.x) {
        const RepSpec& sp = a.spec[t];
        const uint32_t M = (uint32_t)sp.need;
        if (M == 0) continue; // block-uniform
        const uint64_t off = a.offset[t];
        const int64_t top = sp.top;
        const int64_t* sc = a.copy_score + off;
        const int32_t* nd = a.copy_node + off;
        uint32_t* src = a.sort_buf + 2 * off;
        uint32_t* dst = src + M;
        for (uint32_t i = threadIdx.x; i < M; i += REP_THREADS) src[i] = i;
        const uint64_t span = (uint64_t)(top - sp.lo);
        const uint32_t bits = span ? 64u - __clzll((long long)span) : 0u;
        for (uint32_t shift = 0; shift < bits; shift += 8) {
            cta_radix_pass(src, dst, M, [&](uint32_t i) { return (uint32_t)(key(top, sc, t, nd, i) >> shift) & 255u; }, s);
            uint32_t* y = src;
            src = dst;
            dst = y;
        }
        for (uint32_t r = threadIdx.x; r < M; r += REP_THREADS) { // with no pass, thread r wrote src[r] itself
            const uint32_t i = src[r];
            a.out_node[off + r] = nd[i];
            a.out_score[off + r] = sc[i];
        }
        __syncthreads(); // the shared sort state is reused by the next spec
    }
}
__global__ void __launch_bounds__(REP_THREADS) k_rep_order(ReplicaArgs a) {
    rep_order(a, [](int64_t top, const int64_t* sc, uint32_t, const int32_t*, uint32_t i) { return (uint64_t)(top - sc[i]); });
}
// MOST_ALLOCATED: the key is top - s_n(0) of the copy's node
__global__ void __launch_bounds__(REP_THREADS) k_rep_order_most(NodeTable nt, ReplicaArgs a) {
    rep_order(a, [&](int64_t top, const int64_t*, uint32_t t, const int32_t* nd, uint32_t i) {
        const int32_t n = nd[i];
        return (uint64_t)(top - most_alloc_int(nt.free_cpu[n], nt.free_mem[n], nt.alloc_cpu[n], nt.alloc_mem[n],
                                               a.req_cpu[t], a.req_mem[t]));
    });
}

// LEAST_BALANCED: one CTA per spec places its `need' copies one at a time, exactly as step 2 of ks_place_replicas
// defines them.  The whole CTA fills the node scores and the block maxima; then warp 0 alone runs the copies (no CTA
// barrier per copy): the argmax over the block maxima (ties to the lower block, and inside a block to the lower node),
// the copy written at its place, the node advanced to its next copy or retired, and its block's maximum rescanned.
template <int W>
__global__ void __launch_bounds__(REP_THREADS) k_rep_seq(NodeTable nt, ReplicaArgs a, ReplicaSeqArgs q) {
    constexpr int POL = KS_SCORE_LEAST_BALANCED;
    __shared__ int64_t s_best[REP_SEQ_BLOCKS];
    __shared__ int32_t s_node[REP_SEQ_BLOCKS];
    const uint32_t N = nt.N, B = q.block, nb = (N + B - 1) / B;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t* score = q.score + (uint64_t)blockIdx.x * N;
    uint32_t* placed = q.placed + (uint64_t)blockIdx.x * N;
    // the best node of block b, every lane of the calling warp ends with it
    auto block_max = [&](uint32_t b, int64_t& key, int32_t& idx) {
        key = INT64_MIN;
        idx = -1;
        const uint32_t n1 = min(N, (b + 1) * B);
        for (uint32_t n = b * B + lane; n < n1; n += 32) { // ascending n per lane: strict '>' keeps the lowest index
            const int64_t v = score[n];
            if (v > key) {
                key = v;
                idx = (int32_t)n;
            }
        }
        warp_argmax(key, idx);
    };
    for (uint32_t t = blockIdx.x; t < a.T; t += gridDim.x) {
        const uint64_t need = a.spec[t].need;
        if (!need) continue; // block-uniform; k_rep_init wrote the row
        const int64_t rc = a.req_cpu[t], rm = a.req_mem[t];
        uint64_t sel[W];
#pragma unroll
        for (int w = 0; w < W; w++) sel[w] = a.sel[(uint64_t)t * W + w];
        const uint32_t R = a.replicas[t];
        for (uint32_t n = threadIdx.x; n < N; n += REP_THREADS) {
            RepNode v;
            uint64_t cn;
            rep_node<W, POL>(nt, n, rc, rm, sel, R, v, cn);
            score[n] = v.k ? rep_score<POL>(v, rc, rm, 0) : INT64_MIN;
            placed[n] = 0;
        }
        __syncthreads();
        for (uint32_t b = warp; b < nb; b += REP_WARPS) {
            int64_t key;
            int32_t idx;
            block_max(b, key, idx);
            if (lane == 0) {
                s_best[b] = key;
                s_node[b] = idx;
            }
        }
        __syncthreads();
        if (warp == 0) {
            const uint64_t off = a.offset[t];
            uint32_t nodes = 0, most = 0;
            int64_t last = 0;
            for (uint64_t r = 0; r < need; r++) {
                int64_t key = INT64_MIN;
                int32_t bb = -1;
                for (uint32_t b = lane; b < nb; b += 32) // ascending b per lane: strict '>' keeps the lowest block
                    if (s_node[b] >= 0 && s_best[b] > key) {
                        key = s_best[b];
                        bb = (int32_t)b;
                    }
                warp_argmax(key, bb); // blocks are node ranges in order: the lower block holds the lower node
                const int32_t n = s_node[bb];
                if (lane == 0) {
                    if (a.out_node) {
                        a.out_node[off + r] = n;
                        a.out_score[off + r] = key;
                    }
                    const uint32_t j = placed[n] + 1; // copies on n with this one
                    placed[n] = j;
                    nodes += j == 1;
                    most = max(most, j);
                    last = key;
                    RepNode v;
                    uint64_t cn;
                    rep_node<W, POL>(nt, (uint32_t)n, rc, rm, sel, R, v, cn);
                    score[n] = j < v.k ? rep_score<POL>(v, rc, rm, j) : INT64_MIN;
                }
                __syncwarp(); // lane 0's stores to score[] are seen by the rescan
                int64_t k2;
                int32_t i2;
                block_max((uint32_t)bb, k2, i2);
                if (lane == 0) {
                    s_best[bb] = k2;
                    s_node[bb] = i2;
                }
                __syncwarp();
            }
            if (lane == 0) {
                a.rows[t].nodes = nodes;
                a.rows[t].max_per_node = most;
                a.rows[t].last_score = last;
            }
        }
        __syncthreads(); // the scratch and the block maxima are reused by the next spec
    }
}

template <int W, int POL>
static cudaError_t rep_sequence(const NodeTable& nt, const ReplicaArgs& a, cudaStream_t st) {
    const dim3 grid(a.n_chunks, a.T);
    const uint32_t per_spec = (a.T + 127) / 128;
    k_rep_scan<W, POL><<<grid, REP_THREADS, 0, st>>>(nt, a);
    k_rep_init<<<per_spec, 128, 0, st>>>(a);
    for (int i = 0; i < REP_PASSES; i++) {
        k_rep_count<W, POL><<<grid, REP_THREADS, 0, st>>>(nt, a);
        k_rep_narrow<<<per_spec, 128, 0, st>>>(a);
    }
    k_rep_tally<W, POL><<<grid, REP_THREADS, 0, st>>>(nt, a);
    k_rep_settle<<<per_spec, 128, 0, st>>>(a);
    k_rep_emit<W, POL><<<grid, REP_THREADS, 0, st>>>(nt, a);
    g_launches += 5 + 2 * REP_PASSES;
    if (a.out_node) {
        if (POL == KS_SCORE_MOST_ALLOCATED) k_rep_order_most<<<a.T, REP_THREADS, 0, st>>>(nt, a);
        else k_rep_order<<<a.T, REP_THREADS, 0, st>>>(a);
        g_launches++;
    }
    return cudaGetLastError();
}

// LEAST_BALANCED: the scan and the rows, then the copies one at a time
template <int W>
static cudaError_t rep_one_by_one(const NodeTable& nt, const ReplicaArgs& a, const ReplicaSeqArgs& q, cudaStream_t st) {
    constexpr int POL = KS_SCORE_LEAST_BALANCED;
    k_rep_scan<W, POL><<<dim3(a.n_chunks, a.T), REP_THREADS, 0, st>>>(nt, a);
    k_rep_init<<<(a.T + 127) / 128, 128, 0, st>>>(a);
    k_rep_seq<W><<<q.ctas, REP_THREADS, 0, st>>>(nt, a, q);
    g_launches += 3;
    return cudaGetLastError();
}

cudaError_t launch_replicas(const NodeTable& nt, int policy, const ReplicaArgs& a, const ReplicaSeqArgs& q,
                            cudaStream_t st) {
    if (a.T == 0 || nt.N == 0) return cudaSuccess;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W_ = decltype(w)::value;
        return with_policy(policy, [&](auto pol) {
            constexpr int POL = decltype(pol)::value;
            // copy scores can rise and fall under LEAST_BALANCED: no threshold search, the copies go one at a time
            if constexpr (POL == KS_SCORE_LEAST_BALANCED) return rep_one_by_one<W_>(nt, a, q, st);
            else return rep_sequence<W_, POL>(nt, a, st);
        });
    });
}

} // namespace ks
