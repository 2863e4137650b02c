// ks_spread.cu — topology spread for replica placement (ks_place_replicas_spread and, over several keys,
// ks_place_replicas_spread_multi, include/ksched.h; DESIGN.md 5k and 5l), sm_90a.
// The skew rule makes placement sequential: every copy can raise the domain minimum m and change which domains are
// admitted.  So the copies go one at a time, exactly as defined, for every policy:
//   k_spread_order  once per call, one CTA per key: the nodes with a domain sorted stably by domain (ks_sort.cuh's radix pass:
//                   histogram, scan, stable scatter per 8-bit digit), so that inside a domain nodes stay in ascending
//                   index; perm[], each node's position pos[] and the domain starts dstart[D + 1];
//   k_spread_seq    one CTA per spec, specs strided over a grid sized by a scratch budget.  The whole CTA scores the
//                   nodes (s_n(0), INT64_MIN where c_n = 0) and builds three levels of maxima, each a (score, node) key:
//                   node blocks of at most 1024 consecutive positions inside one domain, each domain's best over its
//                   blocks, and groups of 1024 domains, whose maximum counts only the domains the rule admits.  Warp 0
//                   then runs the copies without CTA barriers: the argmax over the groups, the copy, and a rescan of the
//                   node's block, its domain and its group.  When the last eligible domain at m takes a copy, m rises
//                   by one and every group is rescanned (at most final m - initial m times).
// Domain-major order breaks k_rep_seq's "the lower block holds the lower node", so the domain and group levels compare
// (score descending, node ascending) explicitly.
#include "ks_launch.h"
#include "ks_replicas.cuh"
#include "ks_sort.cuh"

namespace ks {

constexpr uint32_t SPREAD_BLOCK = 1024; // nodes per block maximum
constexpr uint32_t SPREAD_GROUP = 1024; // domains per group maximum
constexpr uint32_t SPREAD_GROUPS = (KS_SPREAD_MAX_DOMAINS + SPREAD_GROUP - 1) / SPREAD_GROUP;
constexpr uint64_t SPREAD_BUDGET = 64ull << 20; // scratch of all k_spread_seq CTAs of a call (at least one CTA's)
static_assert(REP_THREADS == SORT_THREADS, "k_spread_order uses ks_sort.cuh's 256-thread radix pass");

// Block slots: block j of domain d is slot d + dstart[d] / 1024 + j.  Domain d's ceil(len / 1024) blocks end at most at
// slot d + 1 + dstart[d + 1] / 1024, where domain d + 1's begin, so the slots are distinct and below D + N / 1024 + 1.
__host__ __device__ __forceinline__ uint64_t spread_slots(uint32_t N, uint32_t D) { return (uint64_t)D + N / SPREAD_BLOCK + 1; }

// Per-CTA scratch, laid out as [score N | block key S | domain key D | placed N | block node S | cnt D | domain node D |
// eligible D] with S = spread_slots(N, D): 8-byte arrays first, and a 16-byte multiple per CTA, so every array is aligned.
__host__ __device__ __forceinline__ uint64_t spread_cta_bytes(uint32_t N, uint32_t D) {
    return (12ull * N + 12ull * spread_slots(N, D) + 20ull * D + 15) & ~15ull;
}

// With K >= 2, the secondaries' state follows in each CTA's scratch: [SpreadSec | stamp S | cnt_i D_i, elig_i D_i for
// each secondary i].  SpreadSec holds each key's m, its number of eligible domains at m, |E|, whether minDomains holds
// m at 0, and lim = m + max_skew (the key admits a domain while its count is below lim); stamp[] marks the block slots
// already rescanned in the current event.
struct SpreadSec {
    uint64_t lim[KS_SPREAD_MAX_KEYS];
    uint32_t m[KS_SPREAD_MAX_KEYS], nmin[KS_SPREAD_MAX_KEYS], n_elig[KS_SPREAD_MAX_KEYS], forced[KS_SPREAD_MAX_KEYS];
};

uint64_t spread_cta_bytes_keys(uint32_t N, const uint32_t* Dk, uint32_t K) {
    uint64_t b = spread_cta_bytes(N, Dk[0]);
    if (K < 2) return b;
    uint64_t sec = sizeof(SpreadSec) + 4ull * spread_slots(N, Dk[0]);
    for (uint32_t i = 1; i < K; i++) sec += 8ull * Dk[i];
    return b + ((sec + 15) & ~15ull);
}

void spread_seq_grid(uint64_t cta_bytes, uint32_t T, int sms, uint32_t* ctas, uint64_t* bytes) {
    const uint64_t fit = std::max<uint64_t>(1, SPREAD_BUDGET / cta_bytes);
    *ctas = (uint32_t)std::min<uint64_t>(std::min<uint64_t>(fit, std::max(T, 1u)), 2ull * (uint64_t)std::max(sms, 1));
    *bytes = *ctas * cta_bytes;
}

// One CTA per key: sort key = the node's domain, D for a node without one (those sort last and are dropped).
__global__ void __launch_bounds__(REP_THREADS) k_spread_order(SpreadOrders os, uint32_t N) {
    __shared__ SortShared s;
    SpreadOrder o = os.key[0];
#pragma unroll
    for (uint32_t k = 1; k < KS_SPREAD_MAX_KEYS; k++)
        if (blockIdx.x == k) o = os.key[k];
    const uint32_t D = o.D;
    const int32_t* dom = o.node_domain;
    auto key = [&](uint32_t n) { return dom[n] < 0 ? D : (uint32_t)dom[n]; };
    uint32_t* src = o.sort_buf;
    uint32_t* dst = src + N;
    for (uint32_t i = threadIdx.x; i < N; i += REP_THREADS) src[i] = i;
    __syncthreads();
    const uint32_t bits = 32u - __clz((int)D); // keys lie in [0, D]
    for (uint32_t shift = 0; shift < bits; shift += 8) {
        cta_radix_pass(src, dst, N, [&](uint32_t n) { return (key(n) >> shift) & 255u; }, s);
        uint32_t* y = src;
        src = dst;
        dst = y;
    }
    // dstart[d'] = p for every d' in (key at p - 1, key at p], with key N -> D: each of 0..D written once
    for (uint32_t p = threadIdx.x; p <= N; p += REP_THREADS) {
        const uint32_t k = p < N ? key(src[p]) : D;
        const int64_t prev = p > 0 ? (int64_t)key(src[p - 1]) : -1;
        for (int64_t d = prev + 1; d <= (int64_t)min(k, D); d++) o.dstart[d] = p;
        if (p < N) {
            o.perm[p] = src[p];
            o.pos[src[p]] = p;
        }
    }
}

// A (score, node) key: larger score first, then lower node; node < 0 = none.
struct SpreadKey {
    int64_t key;
    int32_t node;
};

// MULTI (K >= 2 keys, ks_place_replicas_spread_multi): the structure above is built over the primary key; a node that
// a secondary key refuses counts as INT64_MIN in its block.  A secondary domain reaching lim refuses its nodes, and a
// rise of a secondary's m readmits the domains at the new lim - 1: either way the primary blocks holding those nodes are
// rescanned, each once per event, with their domains and groups.  MULTI = false is the single-key kernel unchanged.
template <int W, int POL, bool MULTI>
__global__ void __launch_bounds__(REP_THREADS) k_spread_seq(NodeTable nt, ReplicaArgs a, SpreadArgs q, SpreadKeys mk) {
    __shared__ int64_t s_gkey[SPREAD_GROUPS];
    __shared__ int32_t s_gnode[SPREAD_GROUPS];
    __shared__ uint64_t red[REP_WARPS];
    __shared__ uint32_t s_row[4]; // warp 0's placed, nodes, most, m after the copies
    __shared__ int64_t s_last;
    const uint32_t N = nt.N, D = q.D, Ne = q.dstart[D];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t S = spread_slots(N, D);
    const uint32_t ng = (D + SPREAD_GROUP - 1) / SPREAD_GROUP;
    unsigned char* base = q.scratch + (uint64_t)blockIdx.x * (MULTI ? mk.cta_bytes : spread_cta_bytes(N, D));
    int64_t* score = reinterpret_cast<int64_t*>(base); // by position
    int64_t* bkey = score + N;
    int64_t* dkey = bkey + S;
    uint32_t* placed = reinterpret_cast<uint32_t*>(dkey + D); // by position
    int32_t* bnode = reinterpret_cast<int32_t*>(placed + N);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(bnode + S);
    int32_t* dnode = reinterpret_cast<int32_t*>(cnt + D);
    uint32_t* elig = reinterpret_cast<uint32_t*>(dnode + D);
    const uint32_t* dstart = q.dstart;
    // MULTI: per internal key i, its counts and eligible flags (key 0's are cnt and elig)
    SpreadSec* sec = nullptr;
    uint32_t* stamp = nullptr;
    uint32_t* kcnt[KS_SPREAD_MAX_KEYS] = {};
    uint32_t* kelig[KS_SPREAD_MAX_KEYS] = {};
    if constexpr (MULTI) {
        sec = reinterpret_cast<SpreadSec*>(base + spread_cta_bytes(N, D));
        stamp = reinterpret_cast<uint32_t*>(sec + 1);
        uint32_t* x = stamp + S;
        kcnt[0] = cnt;
        kelig[0] = elig;
#pragma unroll
        for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
            kcnt[i] = x;
            kelig[i] = x + mk.Dk[i];
            x += 2 * mk.Dk[i]; // 0 past K
        }
    }
    // MULTI: every secondary admits node n
    auto sec_ok = [&](uint32_t n) {
#pragma unroll
        for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++)
            if (i < (int)mk.K && (uint64_t)kcnt[i][mk.dom[i][n]] >= sec->lim[i]) return false;
        return true;
    };

    // the best node of block j of domain d (positions ascending = nodes ascending: strict '>' keeps the lowest), every
    // lane of the calling warp ends with it
    auto block_max = [&](uint32_t d, uint32_t j) {
        SpreadKey r{INT64_MIN, -1};
        const uint32_t p0 = dstart[d] + j * SPREAD_BLOCK, p1 = min(dstart[d + 1], p0 + SPREAD_BLOCK);
        for (uint32_t p = p0 + lane; p < p1; p += 32) {
            const int64_t v = score[p];
            if (v > r.key) {
                if constexpr (MULTI)
                    if (!sec_ok(q.perm[p])) continue;
                r.key = v;
                r.node = (int32_t)q.perm[p];
            }
        }
        warp_argmax(r.key, r.node);
        return r;
    };
    // domain d's best over its block maxima (blocks ascending = nodes ascending)
    auto domain_max = [&](uint32_t d) {
        SpreadKey r{INT64_MIN, -1};
        const uint32_t nb = (dstart[d + 1] - dstart[d] + SPREAD_BLOCK - 1) / SPREAD_BLOCK;
        const uint64_t b0 = d + dstart[d] / SPREAD_BLOCK;
        for (uint32_t j = lane; j < nb; j += 32)
            if (bnode[b0 + j] >= 0 && bkey[b0 + j] > r.key) {
                r.key = bkey[b0 + j];
                r.node = bnode[b0 + j];
            }
        warp_argmax(r.key, r.node);
        return r;
    };
    for (uint32_t t = blockIdx.x; t < a.T; t += gridDim.x) {
        const int64_t rc = a.req_cpu[t], rm = a.req_mem[t];
        uint64_t sel[W];
#pragma unroll
        for (int w = 0; w < W; w++) sel[w] = a.sel[(uint64_t)t * W + w];
        const uint32_t R = a.replicas[t];
        // spec t's entry of the primary in max_skew and min_domains: [T] with one key, [T * K] with several
        const auto tk = [&]() {
            if constexpr (MULTI) return (uint64_t)t * mk.K + mk.col[0];
            else return t;
        }();
        const uint64_t skew = q.max_skew[tk];
        const uint32_t* ex = q.existing ? q.existing + (MULTI ? (uint64_t)t * mk.S + mk.off[0] : (uint64_t)t * D) : nullptr;
        for (uint32_t d = threadIdx.x; d < D; d += REP_THREADS) {
            cnt[d] = ex ? ex[d] : 0u;
            elig[d] = 0;
        }
        if constexpr (MULTI) {
#pragma unroll
            for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                const uint32_t* exi = q.existing ? q.existing + (uint64_t)t * mk.S + mk.off[i] : nullptr;
                for (uint32_t d = threadIdx.x; d < mk.Dk[i]; d += REP_THREADS) {
                    kcnt[i][d] = exi ? exi[d] : 0u;
                    kelig[i][d] = 0;
                }
            }
            for (uint64_t b = threadIdx.x; b < S; b += REP_THREADS) stamp[b] = 0;
        }
        __syncthreads();
        for (uint32_t p = threadIdx.x; p < Ne; p += REP_THREADS) {
            const uint32_t n = q.perm[p];
            RepNode v;
            uint64_t cn;
            rep_node<W, POL>(nt, n, rc, rm, sel, R, v, cn);
            score[p] = v.k ? rep_score<POL>(v, rc, rm, 0) : INT64_MIN;
            placed[p] = 0;
            uint64_t miss = 0;
#pragma unroll
            for (int w = 0; w < W; w++) miss |= sel[w] & ~nt.labels[(uint64_t)w * nt.Npad + n];
            if constexpr (MULTI) { // eligible only with every key; a node without one is never chosen
                bool all = true;
#pragma unroll
                for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) all &= i >= (int)mk.K || mk.dom[i][n] >= 0;
                if (!all) score[p] = INT64_MIN;
                if (!miss && all) {
                    elig[q.node_domain[n]] = 1;
#pragma unroll
                    for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++)
                        if (i < (int)mk.K) kelig[i][mk.dom[i][n]] = 1;
                }
            } else {
                if (!miss) elig[q.node_domain[n]] = 1; // the same value from every writer
            }
        }
        __syncthreads();
        if constexpr (MULTI) { // each secondary's |E|, m and lim; thread 0 publishes them in sec
#pragma unroll
            for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                if (i >= (int)mk.K) break;
                uint64_t ne = 0, lo_i = ~0ull;
                for (uint32_t d = threadIdx.x; d < mk.Dk[i]; d += REP_THREADS)
                    if (kelig[i][d]) {
                        ne++;
                        lo_i = min(lo_i, (uint64_t)kcnt[i][d]);
                    }
                ne = rep_reduce(ne, [](uint64_t x, uint64_t y) { return x + y; }, red);
                lo_i = rep_reduce(lo_i, [](uint64_t x, uint64_t y) { return min(x, y); }, red);
                if (threadIdx.x == 0) {
                    const uint64_t ti = (uint64_t)t * mk.K + mk.col[i];
                    const bool f = ne < (q.min_domains ? q.min_domains[ti] : 0u);
                    const uint32_t mi = ne == 0 || f ? 0u : (uint32_t)lo_i;
                    sec->m[i] = mi;
                    sec->forced[i] = f;
                    sec->n_elig[i] = (uint32_t)ne;
                    sec->lim[i] = (uint64_t)mi + q.max_skew[ti];
                }
            }
            __syncthreads();
        }
        uint64_t n_elig = 0, lo = ~0ull;
        for (uint32_t d = warp; d < D; d += REP_WARPS) {
            const uint32_t nb = (dstart[d + 1] - dstart[d] + SPREAD_BLOCK - 1) / SPREAD_BLOCK;
            const uint64_t b0 = d + dstart[d] / SPREAD_BLOCK;
            SpreadKey best{INT64_MIN, -1};
            for (uint32_t j = 0; j < nb; j++) {
                const SpreadKey b = block_max(d, j);
                if (lane == 0) {
                    bkey[b0 + j] = b.key;
                    bnode[b0 + j] = b.node;
                }
                if (b.node >= 0 && b.key > best.key) best = b; // blocks in node order: strict '>' keeps the lowest
            }
            if (lane == 0) {
                dkey[d] = best.key;
                dnode[d] = best.node;
                if (elig[d]) {
                    n_elig++;
                    lo = min(lo, (uint64_t)cnt[d]);
                }
            }
        }
        n_elig = rep_reduce(n_elig, [](uint64_t x, uint64_t y) { return x + y; }, red);
        lo = rep_reduce(lo, [](uint64_t x, uint64_t y) { return min(x, y); }, red);
        const uint32_t mind = q.min_domains ? q.min_domains[tk] : 0u;
        const bool forced = n_elig < mind; // minDomains holds m at 0
        uint32_t m = n_elig == 0 || forced ? 0u : (uint32_t)lo;
        // the rule admits domain d while cnt[d] + 1 - m <= skew
        auto admitted = [&](uint32_t d) { return elig[d] && (uint64_t)cnt[d] < (uint64_t)m + skew; };
        // group g's best admitted domain, compared explicitly: domain order is not node order
        auto group_max = [&](uint32_t g) {
            SpreadKey r{INT64_MIN, -1};
            const uint32_t d1 = min(D, (g + 1) * SPREAD_GROUP);
            for (uint32_t d = g * SPREAD_GROUP + lane; d < d1; d += 32) {
                const int32_t dn = dnode[d];
                if (dn >= 0 && admitted(d) && topk_beats(dkey[d], dn, r.key, r.node)) {
                    r.key = dkey[d];
                    r.node = dn;
                }
            }
            warp_argmax(r.key, r.node);
            return r;
        };
        for (uint32_t g = warp; g < ng; g += REP_WARPS) {
            const SpreadKey b = group_max(g);
            if (lane == 0) {
                s_gkey[g] = b.key;
                s_gnode[g] = b.node;
            }
        }
        __syncthreads();
        if (warp == 0) {
            // eligible domains at m; not needed while minDomains holds m at 0
            auto at_min = [&]() {
                uint32_t c = 0;
                for (uint32_t d = lane; d < D; d += 32) c += elig[d] && cnt[d] == m;
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
                return c;
            };
            uint32_t nmin = n_elig && !forced ? at_min() : 0u;
            // MULTI: each secondary's m, eligible domains at m and minDomains flag, the same in every lane
            uint32_t km[KS_SPREAD_MAX_KEYS] = {}, kmin[KS_SPREAD_MAX_KEYS] = {};
            bool kforced[KS_SPREAD_MAX_KEYS] = {};
            uint32_t ev = 0; // the rescan event, for stamp[]
            auto count_at = [&](const uint32_t* el, const uint32_t* cn, uint32_t Dn, uint32_t mv) {
                uint32_t c = 0;
                for (uint32_t d = lane; d < Dn; d += 32) c += el[d] && cn[d] == mv;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
                return c;
            };
            // rescan block jb of primary domain d, then d and its group
            auto refresh = [&](uint32_t d, uint32_t jb) {
                const uint64_t b = d + dstart[d] / SPREAD_BLOCK + jb;
                const SpreadKey nb = block_max(d, jb);
                if (lane == 0) {
                    bkey[b] = nb.key;
                    bnode[b] = nb.node;
                }
                __syncwarp();
                const SpreadKey nd = domain_max(d);
                if (lane == 0) {
                    dkey[d] = nd.key;
                    dnode[d] = nd.node;
                }
                __syncwarp();
                const uint32_t g = d / SPREAD_GROUP;
                const SpreadKey ngk = group_max(g);
                if (lane == 0) {
                    s_gkey[g] = ngk.key;
                    s_gnode[g] = ngk.node;
                }
                __syncwarp();
            };
            // each lane with hit holds node n2 at primary position p2: rescan their blocks, each once per event
            auto touch = [&](bool hit, uint32_t n2, uint32_t p2) {
                uint32_t d1 = 0, jb = 0;
                uint64_t slot = ~0ull;
                if (hit) {
                    d1 = (uint32_t)q.node_domain[n2];
                    jb = (p2 - dstart[d1]) / SPREAD_BLOCK;
                    slot = d1 + dstart[d1] / SPREAD_BLOCK + jb;
                }
                const uint32_t peers = __match_any_sync(0xffffffffu, slot);
                const bool lead = hit && (uint32_t)(__ffs(peers) - 1) == lane && stamp[slot] != ev;
                if (lead) stamp[slot] = ev;
                for (uint32_t todo = __ballot_sync(0xffffffffu, lead); todo; todo &= todo - 1) {
                    const int src = __ffs(todo) - 1;
                    refresh(__shfl_sync(0xffffffffu, d1, src), __shfl_sync(0xffffffffu, jb, src));
                }
            };
            if constexpr (MULTI) {
#pragma unroll
                for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                    if (i >= (int)mk.K) break;
                    km[i] = sec->m[i];
                    kforced[i] = sec->forced[i];
                    kmin[i] = sec->n_elig[i] && !kforced[i] ? count_at(kelig[i], kcnt[i], mk.Dk[i], km[i]) : 0u;
                }
            }
            const uint64_t off = a.offset[t];
            uint32_t r = 0, nodes = 0, most = 0;
            int64_t last = 0;
            for (; n_elig && r < R; r++) {
                SpreadKey b{INT64_MIN, -1};
                for (uint32_t g = lane; g < ng; g += 32)
                    if (topk_beats(s_gkey[g], s_gnode[g], b.key, b.node)) {
                        b.key = s_gkey[g];
                        b.node = s_gnode[g];
                    }
                warp_argmax(b.key, b.node);
                if (b.node < 0) break; // no candidate: the state does not change, no later copy fits either
                const uint32_t n = (uint32_t)b.node, d = (uint32_t)q.node_domain[n], p = q.pos[n];
                uint32_t c_old = 0, j = 0;
                if (lane == 0) {
                    if (a.out_node) {
                        a.out_node[off + r] = b.node;
                        a.out_score[off + r] = b.key;
                    }
                    j = placed[p] + 1; // copies on n with this one
                    placed[p] = j;
                    RepNode v;
                    uint64_t cn;
                    rep_node<W, POL>(nt, n, rc, rm, sel, R, v, cn);
                    score[p] = j < v.k ? rep_score<POL>(v, rc, rm, j) : INT64_MIN;
                    c_old = cnt[d];
                    cnt[d] = c_old + 1;
                }
                j = __shfl_sync(0xffffffffu, j, 0);
                c_old = __shfl_sync(0xffffffffu, c_old, 0);
                nodes += j == 1;
                most = max(most, j);
                last = b.key;
                __syncwarp(); // lane 0's stores to score[] and cnt[] are seen by the rescans
                bool raised = false;
                if (!forced && c_old == m && --nmin == 0) { // the last domain at m took a copy
                    m++;
                    nmin = at_min();
                    raised = true;
                }
                uint32_t refuse = 0, rise = 0; // MULTI: bit i = secondary i refuses d_i(n) / its m rose
                if constexpr (MULTI) {
#pragma unroll
                    for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                        if (i >= (int)mk.K) break;
                        const uint32_t di = (uint32_t)mk.dom[i][n];
                        uint32_t co = 0;
                        if (lane == 0) {
                            co = kcnt[i][di];
                            kcnt[i][di] = co + 1;
                        }
                        co = __shfl_sync(0xffffffffu, co, 0);
                        __syncwarp();
                        if (!kforced[i] && co == km[i] && --kmin[i] == 0) {
                            km[i]++;
                            kmin[i] = count_at(kelig[i], kcnt[i], mk.Dk[i], km[i]);
                            if (lane == 0) sec->lim[i]++;
                            rise |= 1u << i;
                        } else if ((uint64_t)co + 1 == sec->lim[i]) {
                            refuse |= 1u << i;
                        }
                        __syncwarp();
                    }
                }
                const uint32_t jb = (p - dstart[d]) / SPREAD_BLOCK;
                const SpreadKey nb = block_max(d, jb);
                if (lane == 0) {
                    bkey[d + dstart[d] / SPREAD_BLOCK + jb] = nb.key;
                    bnode[d + dstart[d] / SPREAD_BLOCK + jb] = nb.node;
                }
                __syncwarp();
                const SpreadKey nd = domain_max(d);
                if (lane == 0) {
                    dkey[d] = nd.key;
                    dnode[d] = nd.node;
                }
                __syncwarp();
                // a rise of m can admit a domain in every group; otherwise only d's group changed
                for (uint32_t g = raised ? 0u : d / SPREAD_GROUP; g < (raised ? ng : d / SPREAD_GROUP + 1); g++) {
                    const SpreadKey ngk = group_max(g);
                    if (lane == 0) {
                        s_gkey[g] = ngk.key;
                        s_gnode[g] = ngk.node;
                    }
                }
                __syncwarp();
                if constexpr (MULTI) {
#pragma unroll
                    for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                        if (refuse >> i & 1) { // d_i(n) reached lim: its nodes leave their blocks
                            const uint32_t di = (uint32_t)mk.dom[i][n], x1 = mk.kdstart[i][di + 1];
                            ev++;
                            for (uint32_t x = mk.kdstart[i][di]; x < x1; x += 32) {
                                const bool in = x + lane < x1;
                                const uint32_t n2 = in ? mk.kperm[i][x + lane] : 0u, p2 = in ? q.pos[n2] : 0u;
                                touch(in && p2 < Ne, n2, p2);
                            }
                        }
                        if (rise >> i & 1) { // m rose: the domains at the new lim - 1 are admitted again
                            const uint64_t lim = sec->lim[i];
                            ev++;
                            for (uint32_t x = 0; x < Ne; x += 32) {
                                const uint32_t p2 = x + lane, n2 = p2 < Ne ? q.perm[p2] : 0u;
                                const int32_t d2 = p2 < Ne ? mk.dom[i][n2] : -1;
                                touch(d2 >= 0 && (uint64_t)kcnt[i][d2] + 1 == lim, n2, p2);
                            }
                        }
                    }
                }
            }
            if (lane == 0) {
                s_row[0] = r;
                s_row[1] = nodes;
                s_row[2] = most;
                s_row[3] = m;
                s_last = last;
                if constexpr (MULTI) {
                    sec->m[0] = m;
                    sec->lim[0] = (uint64_t)m + skew;
                    sec->n_elig[0] = (uint32_t)n_elig;
#pragma unroll
                    for (int i = 1; i < (int)KS_SPREAD_MAX_KEYS; i++) sec->m[i] = km[i];
                }
            }
        }
        __syncthreads();
        const uint32_t placed_t = s_row[0];
        if constexpr (!MULTI) {
            // the lowest admitted eligible domain: at a stop, every admitted domain holds no further copy
            uint64_t blocked = ~0ull;
            if (placed_t < R) {
                m = s_row[3];
                for (uint32_t d = threadIdx.x; d < D; d += REP_THREADS)
                    if (admitted(d)) blocked = min(blocked, (uint64_t)d);
            }
            blocked = rep_reduce(blocked, [](uint64_t x, uint64_t y) { return min(x, y); }, red);
            if (q.out_count)
                for (uint32_t d = threadIdx.x; d < D; d += REP_THREADS) q.out_count[(uint64_t)t * D + d] = cnt[d];
            if (threadIdx.x == 0) {
                ks_spread_plan row;
                row.placed = placed_t;
                row.nodes = s_row[1];
                row.max_per_node = s_row[2];
                row.eligible_domains = (uint32_t)n_elig;
                row.min_count = s_row[3];
                row.blocked_domain = blocked == ~0ull ? -1 : (int32_t)blocked;
                row.last_score = s_last;
                q.rows[t] = row;
            }
        } else {
            // at a stop, flag 3 marks each key's domains that hold a node with room (score above INT64_MIN: eligible,
            // with j_n < c_n) which every other key admits; blocked = the lowest eligible domain without the mark that
            // the key's own rule admits
            if (placed_t < R) {
                const uint32_t all = (1u << mk.K) - 1;
                for (uint32_t p = threadIdx.x; p < Ne; p += REP_THREADS) {
                    if (score[p] == INT64_MIN) continue;
                    const uint32_t n = q.perm[p];
                    uint32_t ok = 0;
#pragma unroll
                    for (int i = 0; i < (int)KS_SPREAD_MAX_KEYS; i++)
                        if (i < (int)mk.K && (uint64_t)kcnt[i][mk.dom[i][n]] < sec->lim[i]) ok |= 1u << i;
#pragma unroll
                    for (int i = 0; i < (int)KS_SPREAD_MAX_KEYS; i++)
                        if (i < (int)mk.K && (ok | 1u << i) == all) kelig[i][mk.dom[i][n]] = 3; // the same from every writer
                }
                __syncthreads();
            }
#pragma unroll
            for (int i = 0; i < (int)KS_SPREAD_MAX_KEYS; i++) {
                if (i >= (int)mk.K) break;
                uint64_t blocked = ~0ull;
                if (placed_t < R)
                    for (uint32_t d = threadIdx.x; d < mk.Dk[i]; d += REP_THREADS)
                        if (kelig[i][d] == 1 && (uint64_t)kcnt[i][d] < sec->lim[i]) blocked = min(blocked, (uint64_t)d);
                blocked = rep_reduce(blocked, [](uint64_t x, uint64_t y) { return min(x, y); }, red);
                if (q.out_count)
                    for (uint32_t d = threadIdx.x; d < mk.Dk[i]; d += REP_THREADS)
                        q.out_count[(uint64_t)t * mk.S + mk.off[i] + d] = kcnt[i][d];
                if (threadIdx.x == 0) {
                    ks_spread_plan row;
                    row.placed = placed_t;
                    row.nodes = s_row[1];
                    row.max_per_node = s_row[2];
                    row.eligible_domains = sec->n_elig[i];
                    row.min_count = sec->m[i];
                    row.blocked_domain = blocked == ~0ull ? -1 : (int32_t)blocked;
                    row.last_score = s_last;
                    q.rows[(uint64_t)t * mk.K + mk.col[i]] = row;
                }
            }
        }
        __syncthreads(); // the scratch is reused by the next spec
    }
}

cudaError_t launch_spread(const NodeTable& nt, int policy, const ReplicaArgs& a, const SpreadOrders& o,
                          const SpreadArgs& q, const SpreadKeys& mk, cudaStream_t st) {
    if (a.T == 0 || nt.N == 0) return cudaSuccess;
    k_spread_order<<<o.K, REP_THREADS, 0, st>>>(o, nt.N);
    g_launches++;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W_ = decltype(w)::value;
        return with_policy(policy, [&](auto pol) {
            constexpr int POL = decltype(pol)::value;
            if (o.K > 1) k_spread_seq<W_, POL, true><<<q.ctas, REP_THREADS, 0, st>>>(nt, a, q, mk);
            else k_spread_seq<W_, POL, false><<<q.ctas, REP_THREADS, 0, st>>>(nt, a, q, mk);
            g_launches++;
            return cudaGetLastError();
        });
    });
}

} // namespace ks
