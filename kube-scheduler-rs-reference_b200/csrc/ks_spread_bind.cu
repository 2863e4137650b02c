// ks_spread_bind.cu — the bind calls of include/ksched.h: ks_spread_bind (topology spread, DESIGN.md 5m),
// ks_affinity_bind (and inter-pod affinity, 5n), ks_profile_bind (and the soft PodTopologySpread and InterPodAffinity
// scores, 5o), ks_node_bind (and TaintToleration and NodeAffinity, 5p), ks_fit_bind (and the pod count and scalar
// resources of NodeResourcesFit, 5r) and ks_gang_fit_bind (ks_fit_bind with gangs that commit or roll back whole, 5s).
// Each binds a mixed pod queue one pod at a time, each pod against the counts and the free[] every earlier pod left, as
// upstream kube-scheduler runs one scheduling cycle per pod.  The calls differ by one BindMode (ks_launch.h), SPREAD,
// AFFINITY, PROFILE, NODE, FIT (NODE's launches and walk, with the resources) or GANG_FIT (FIT's, with the gangs'
// rollback), and share:
//   BindFilter          the candidate filter: fit and selector, (FIT) the scalar resources, (NODE, FIT) the node's rule
//                       word, hard spread and (AFF, every mode but SPREAD) rules 1-3 of the header
//   k_bind_setup        one CTA per group (grid-strided): the group's eligible domains per constrained key, its counts
//                       (existing, or 0), and per key |E|, m, the number of eligible domains at m and the minDomains flag;
//                       NR (NODE) also drops the nodes that fail the group's required node affinity
//   k_bind_seq          one cooperative launch that walks the pods, shaped like k_gang_batch (ks_stream.cu): every CTA
//                       owns one slice of the node table and grid barriers separate each pod's phases.  SPREAD and
//                       AFFINITY: phase A scans every slice into one partial per CTA, phase B (CTA 0) merges the partials
//                       in CTA order, charges free[], writes the binding and raises the counts.  PROFILE and NODE: three
//                       passes, because the soft scores need grid-wide reductions over the candidates before any node's
//                       total exists, then the same commit.
//   launch_bind         one mode's launches, in order
// Per call, k_affinity_setup and k_profile_setup apply the existing pods' update entries (every mode but SPREAD, and
// PROFILE, NODE and FIT), and k_node_rules_setup writes one rule word per (node-rule class, node) (NODE, FIT).
#include "ks_internal.cuh"
#include "ks_launch.h"

#include <algorithm>
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace ks {

constexpr uint32_t SBD_THREADS = 256;
constexpr uint32_t SBD_WARPS = SBD_THREADS / 32;

// Per (group, key) state words in a.gk: the minimum m, the eligible domains whose count is m, |E| and the flags
enum : uint32_t { GK_M = 0, GK_AT_M = 1, GK_NE = 2, GK_FLAGS = 3, GK_WORDS = 4 };
constexpr uint32_t GK_CONSTRAINED = 1u, GK_FORCED = 2u; // max_skew >= 1; minDomains holds m at 0

// CTA-wide sum and minimum of one value per thread; every thread gets the result.  s holds SBD_WARPS words.
__device__ __forceinline__ uint32_t cta_sum(uint32_t v, uint32_t* s) {
    v = __reduce_add_sync(0xffffffffu, v);
    __syncthreads(); // s is free
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t r = 0;
#pragma unroll
    for (uint32_t w = 0; w < SBD_WARPS; w++) r += s[w];
    return r;
}
__device__ __forceinline__ uint32_t cta_min(uint32_t v, uint32_t* s) {
    v = __reduce_min_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t r = 0xffffffffu;
#pragma unroll
    for (uint32_t w = 0; w < SBD_WARPS; w++) r = min(r, s[w]);
    return r;
}

// The keys group g constrains, one bit per key (max_skew >= 1)
__device__ __forceinline__ uint32_t constrained_keys(const SpreadBindArgs& a, int32_t g) {
    uint32_t ck = 0;
    if (g >= 0)
        for (uint32_t k = 0; k < a.K; k++)
            if (__ldg(a.max_skew + (size_t)g * a.K + k)) ck |= 1u << k;
    return ck;
}

// The eligible domains of key k at count m: the domain count of a (group, key) after its minimum has risen
__device__ __forceinline__ uint32_t domains_at(const SpreadBindArgs& a, uint32_t g, uint32_t k, uint32_t m, uint32_t* s) {
    const size_t base = (size_t)g * a.S + a.Pk[k];
    uint32_t c = 0;
    for (uint32_t d = threadIdx.x; d < a.Dk[k]; d += SBD_THREADS)
        c += a.elig[base + d] && __ldcg(a.cnt + base + d) == m;
    return cta_sum(c, s);
}

// NR (ks_node_bind): a node is also eligible only when it passes the group's required node affinity (the NR_AFF_OK bit
// of its rule word in the group's class row, nrules / ncls of ProfileBindArgs)
template <int W, bool NR>
__device__ __forceinline__ void spread_bind_setup(const SpreadBindArgs& a, const uint32_t* nrules, const uint32_t* ncls) {
    __shared__ uint32_t s_red[SBD_WARPS];
    const uint32_t tid = threadIdx.x;
    for (uint32_t g = blockIdx.x; g < a.G; g += gridDim.x) {
        uint32_t* cnt = a.cnt + (size_t)g * a.S;
        uint8_t* el = a.elig + (size_t)g * a.S;
        for (uint32_t i = tid; i < a.S; i += SBD_THREADS) {
            cnt[i] = a.existing ? __ldg(a.existing + (size_t)g * a.S + i) : 0u;
            el[i] = 0;
        }
        const uint32_t ck = constrained_keys(a, (int32_t)g);
        __syncthreads();
        if (ck) { // eligible: the group's selector matches and the node carries every key the group constrains
            uint64_t sw[W];
#pragma unroll
            for (int w = 0; w < W; w++) sw[w] = __ldg(a.gsel + (size_t)g * W + w);
            const uint32_t* nrow = NR ? nrules + (size_t)__ldg(ncls + g + 1) * a.N : nullptr;
            for (uint32_t n = tid; n < a.N; n += SBD_THREADS) {
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sw[w] & ~__ldg(a.labels + (size_t)w * a.Npad + n);
                if (miss) continue;
                if (NR && !(__ldg(nrow + n) & NR_AFF_OK)) continue;
                int32_t d[KS_SPREAD_MAX_KEYS];
                bool all = true;
#pragma unroll
                for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
                    d[k] = (ck >> k & 1u) ? __ldg(a.dom + (size_t)k * a.N + n) : 0;
                    all &= d[k] >= 0;
                }
                if (!all) continue;
#pragma unroll
                for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
                    if (ck >> k & 1u) el[a.Pk[k] + (uint32_t)d[k]] = 1;
            }
        }
        __syncthreads();
        for (uint32_t k = 0; k < a.K; k++) {
            uint32_t* st = a.gk + ((size_t)g * a.K + k) * GK_WORDS;
            if (!(ck >> k & 1u)) {
                if (tid < GK_WORDS) st[tid] = 0;
                continue;
            }
            uint32_t ne = 0, mn = 0xffffffffu;
            for (uint32_t d = tid; d < a.Dk[k]; d += SBD_THREADS)
                if (el[a.Pk[k] + d]) {
                    ne++;
                    mn = min(mn, cnt[a.Pk[k] + d]);
                }
            ne = cta_sum(ne, s_red);
            mn = cta_min(mn, s_red);
            const uint32_t mind = a.min_domains ? __ldg(a.min_domains + (size_t)g * a.K + k) : 0u;
            const bool forced = ne < mind; // upstream's minDomains: the global minimum counts as 0
            const uint32_t m = ne == 0 || forced ? 0u : mn;
            const uint32_t at = ne == 0 || forced ? 0u : domains_at(a, g, k, m, s_red);
            if (tid == 0) {
                st[GK_M] = m;
                st[GK_AT_M] = at;
                st[GK_NE] = ne;
                st[GK_FLAGS] = GK_CONSTRAINED | (forced ? GK_FORCED : 0u);
            }
        }
        __syncthreads(); // el and cnt of this group are final before the CTA's next group
    }
}

template <int W, bool NR>
__global__ void __launch_bounds__(SBD_THREADS) k_bind_setup(const ProfileBindArgs a) {
    spread_bind_setup<W, NR>(a.b, a.nrules, a.ncls);
}

// Inter-pod affinity: one update entry of a pod bound at node n.  Entries of one list name distinct (group, key, kind)
// arrays, so CTA 0's threads raise them without atomics; the existing pods' lists run concurrently and use atomics.
template <bool ATOMIC>
__device__ __forceinline__ void affinity_raise(const SpreadBindArgs& a, uint32_t entry, uint32_t n) {
    const uint32_t h = entry & 0xffffu, k = entry >> 16 & 0xfu, kind = entry >> 20;
    const int32_t d = __ldg(a.dom + (size_t)k * a.N + n);
    if (d < 0) return; // the node lacks the key: no domain to count in
    uint32_t* c = a.acnt + __ldg(a.abase + ((size_t)h * a.K + k) * 2 + kind) + (uint32_t)d;
    if (ATOMIC) atomicAdd(c, 1u);
    else *c = __ldcg(c) + 1;
    if (kind) a.acnt[a.any_base + h] = 1; // a pod of M_h sits on a node that carries one of h's affinity keys
}

// The candidate filter of every bind walk for pod p: fit, selector and, for a constrained pod, cnt < m + max_skew on
// every constrained key (the bound formed once per pod); AFF: then rules 1-3 of ks_affinity_bind against the pod's
// group's counter bases and first-pod flag, formed once per pod.  Without AFF (ks_spread_bind, whose abase, aflag and
// acnt are NULL) none of them is read.  FIT (ks_fit_bind): after fit and selector, the scalar resources the pod requests,
// their mask and amounts formed once per pod; the other instances read none of it.
template <int W, bool AFF, bool FIT = false>
struct BindFilter {
    int32_t g;
    int64_t rc, rm;
    uint64_t sw[W];
    uint32_t ck;
    uint64_t lim[KS_SPREAD_MAX_KEYS];
    const uint32_t* cnt;
    uint32_t bB[KS_SPREAD_MAX_KEYS], bA[KS_SPREAD_MAX_KEYS]; // AFF: B_{g,k} / A_{g,k} bases, AFF_NONE = no such array
    bool first;                                              // AFF: upstream's first-pod rule holds for g
    uint32_t rmask;                                          // FIT: bit r = the pod requests resource r
    int64_t rreq[KS_BIND_MAX_RESOURCES];                     // FIT: its requests
    const int64_t* rfree;                                    // FIT: free_r[n] at r * N + n

    __device__ __forceinline__ BindFilter(const ProfileBindArgs& q, uint32_t p) : BindFilter(q.b, p) {
        if constexpr (FIT) {
            rmask = 0;
            rfree = q.res_free;
#pragma unroll
            for (uint32_t r = 0; r < KS_BIND_MAX_RESOURCES; r++) {
                rreq[r] = r < q.R ? __ldg(q.res_req + (size_t)p * q.R + r) : 0;
                if (rreq[r]) rmask |= 1u << r;
            }
        }
    }

    __device__ __forceinline__ BindFilter(const SpreadBindArgs& a, uint32_t p) {
        g = __ldg(a.group + p);
        rc = __ldg(a.req_cpu + p);
        rm = __ldg(a.req_mem + p);
#pragma unroll
        for (int w = 0; w < W; w++) sw[w] = __ldg(a.sel + (size_t)p * W + w);
        ck = constrained_keys(a, g);
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
            lim[k] = (ck >> k & 1u) ? (uint64_t)__ldcg(a.gk + ((size_t)g * a.K + k) * GK_WORDS + GK_M) +
                                          __ldg(a.max_skew + (size_t)g * a.K + k)
                                    : 0;
            if constexpr (AFF) {
                const bool on = g >= 0 && k < a.K;
                bB[k] = on ? __ldg(a.abase + ((size_t)g * a.K + k) * 2) : AFF_NONE;
                bA[k] = on ? __ldg(a.abase + ((size_t)g * a.K + k) * 2 + 1) : AFF_NONE;
            }
        }
        cnt = a.cnt + (size_t)(g < 0 ? 0 : g) * a.S;
        if constexpr (AFF) first = g >= 0 && (__ldg(a.aflag + g) & AFF_SELF) && __ldcg(a.acnt + a.any_base + g) == 0;
    }
    // 0: unfit (fit or selector), 1: refused by spread, 2: refused by rules 1-3 (AFF), 3: candidate; NR (ks_node_bind)
    // with the node's rule word rw: 4: refused by a taint, 5: refused by required node affinity, both before spread;
    // FIT: 6: refused by a scalar resource, before the taints
    template <bool NR = false>
    __device__ __forceinline__ int test(const SpreadBindArgs& a, uint32_t n, int64_t fc, int64_t fm,
                                        uint32_t rw = 0) const {
        uint64_t miss = 0;
#pragma unroll
        for (int w = 0; w < W; w++) miss |= sw[w] & ~__ldg(a.labels + (size_t)w * a.Npad + n);
        if (!(rc <= fc && rm <= fm && miss == 0)) return 0;
        if constexpr (FIT) {
            bool fits = true;
#pragma unroll
            for (uint32_t r = 0; r < KS_BIND_MAX_RESOURCES; r++)
                if (rmask >> r & 1u) fits &= rreq[r] <= __ldcg(rfree + (size_t)r * a.N + n);
            if (!fits) return 6;
        }
        if (NR && (rw & NR_REASON)) return 3 + (int)(rw & NR_REASON);
        bool ok = true;
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
            if (ck >> k & 1u) {
                const int32_t d = __ldg(a.dom + (size_t)k * a.N + n);
                ok &= d >= 0 && __ldcg(cnt + a.Pk[k] + (uint32_t)max(d, 0)) < lim[k];
            }
        if (!ok) return 1;
        bool aok = true;
        if constexpr (AFF) {
#pragma unroll
            for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
                if ((bB[k] & bA[k]) != AFF_NONE) {
                    const int32_t d = __ldg(a.dom + (size_t)k * a.N + n);
                    const uint32_t dd = (uint32_t)max(d, 0);
                    if (bB[k] != AFF_NONE) aok &= d < 0 || __ldcg(a.acnt + bB[k] + dd) == 0;        // rules 1 and 2
                    if (bA[k] != AFF_NONE) aok &= d >= 0 && (first || __ldcg(a.acnt + bA[k] + dd) > 0); // rule 3
                }
        }
        return aok ? 3 : 2;
    }
};

// Phase A of pod p in this CTA's slice [n0, n1): the filter; the best candidate by the policy's key (ties to the lower
// node) and the spread refusals into the CTA's partial, AFF also the refusals of rules 1-3 (s_aref / paref).
template <int W, bool AFF>
__device__ __forceinline__ void spread_bind_scan(const SpreadBindArgs& a, uint32_t p, uint32_t n0, uint32_t n1,
                                                 int64_t* s_key, int32_t* s_idx, uint32_t* s_ref, uint32_t* s_aref) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const BindFilter<W, AFF> f(a, p);
    int64_t best = INT64_MIN;
    int32_t bidx = -1;
    uint32_t refused = 0, arefused = 0;
    for (uint32_t n = n0 + tid; n < n1; n += SBD_THREADS) {
        const int64_t fc = __ldcg(a.free_cpu + n), fm = __ldcg(a.free_mem + n);
        const int r = f.test(a, n, fc, fm);
        refused += r == 1;
        if constexpr (AFF) arefused += r == 2;
        if (r != 3) continue;
        const int64_t key = alloc_score_rt(a.policy, fc, fm, a.alloc_cpu, a.alloc_mem, n, f.rc, f.rm);
        if (key > best) { // ascending n per thread: strict '>' keeps the lowest index
            best = key;
            bidx = (int32_t)n;
        }
    }
    warp_argmax(best, bidx);
    refused = __reduce_add_sync(0xffffffffu, refused);
    if constexpr (AFF) arefused = __reduce_add_sync(0xffffffffu, arefused);
    if (lane == 0) {
        s_key[warp] = best;
        s_idx[warp] = bidx;
        s_ref[warp] = refused;
        if constexpr (AFF) s_aref[warp] = arefused;
    }
    __syncthreads();
    if (warp == 0) {
        best = lane < SBD_WARPS ? s_key[lane] : INT64_MIN;
        bidx = lane < SBD_WARPS ? s_idx[lane] : -1;
        warp_argmax(best, bidx);
        refused = __reduce_add_sync(0xffffffffu, lane < SBD_WARPS ? s_ref[lane] : 0u);
        if constexpr (AFF) arefused = __reduce_add_sync(0xffffffffu, lane < SBD_WARPS ? s_aref[lane] : 0u);
        if (lane == 0) {
            a.pkey[blockIdx.x] = best;
            a.pidx[blockIdx.x] = bidx;
            a.pref[blockIdx.x] = refused;
            if constexpr (AFF) a.paref[blockIdx.x] = arefused;
        }
    }
}

// Phase B of pod p, CTA 0 only: merge the partials in CTA order, write the binding, charge free[] and raise the group's
// counts.  When the last eligible domain at m takes the pod, m rises by exactly one and the domains at the new m are
// counted over the group's domains of that key (the counts only rise, so at most final m - initial m such passes).
// The refusals go to out_refused[R * p + O] at the mode's stride R and offset O: 1 / 0 for SPREAD, 2 / 0 for AFFINITY
// and PROFILE (spread, then affinity), 4 / 2 for NODE (after the taint and node-affinity words of profile_commit), 5 / 3
// for FIT (after the resource word and the two node-rule words).  AFF: the bound pod's update entries across the CTA
// (s_bidx).
template <BindMode M>
__device__ __forceinline__ void spread_bind_commit(const SpreadBindArgs& a, uint32_t p, uint32_t* s_rescan,
                                                   uint32_t* s_red, int32_t* s_bidx) {
    constexpr bool AFF = M != BIND_SPREAD;
    constexpr size_t R = bind_refusal_words(M), O = M == BIND_FIT ? 3 : M == BIND_NODE ? 2 : 0;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const int32_t g = __ldg(a.group + p);
    if (tid < 32) {
        int64_t best = INT64_MIN;
        int32_t bidx = -1;
        uint32_t refused = 0, arefused = 0;
        for (uint32_t c = lane; c < gridDim.x; c += 32) { // ascending CTA = ascending node range
            merge_partial(best, bidx, __ldcg(a.pkey + c), __ldcg(a.pidx + c));
            refused += __ldcg(a.pref + c);
            if constexpr (AFF) arefused += __ldcg(a.paref + c);
        }
        warp_argmax(best, bidx);
        refused = __reduce_add_sync(0xffffffffu, refused);
        if constexpr (AFF) arefused = __reduce_add_sync(0xffffffffu, arefused);
        if (lane == 0) {
            uint32_t rescan = 0;
            a.out_idx[p] = bidx;
            a.out_score[p] = bidx >= 0 ? key_score_rt(a.policy, best, a.req_cpu, a.req_mem, p) : 0;
            a.out_refused[R * p + O] = refused;
            if constexpr (AFF) {
                a.out_refused[R * p + O + 1] = arefused;
                *s_bidx = bidx;
            }
            if (bidx >= 0) {
                a.free_cpu[bidx] = __ldcg(a.free_cpu + bidx) - __ldg(a.req_cpu + p);
                a.free_mem[bidx] = __ldcg(a.free_mem + bidx) - __ldg(a.req_mem + p);
                const uint32_t ck = constrained_keys(a, g);
                for (uint32_t k = 0; k < a.K; k++) {
                    if (!(ck >> k & 1u)) continue;
                    const uint32_t d = (uint32_t)__ldg(a.dom + (size_t)k * a.N + bidx);
                    uint32_t* c = a.cnt + (size_t)g * a.S + a.Pk[k] + d;
                    const uint32_t before = __ldcg(c);
                    *c = before + 1;
                    uint32_t* st = a.gk + ((size_t)g * a.K + k) * GK_WORDS;
                    if ((__ldcg(st + GK_FLAGS) & GK_FORCED) || before != __ldcg(st + GK_M)) continue;
                    const uint32_t at = __ldcg(st + GK_AT_M) - 1;
                    st[GK_AT_M] = at;
                    if (at == 0) { // the last domain at m took the pod: m + 1, and its domains are counted below
                        st[GK_M] = before + 1;
                        rescan |= 1u << k;
                    }
                }
            }
            *s_rescan = rescan;
        }
    }
    __syncthreads();
    const uint32_t rescan = *s_rescan;
    for (uint32_t k = 0; k < a.K; k++) {
        if (!(rescan >> k & 1u)) continue;
        uint32_t* st = a.gk + ((size_t)g * a.K + k) * GK_WORDS;
        const uint32_t at = domains_at(a, (uint32_t)g, k, __ldcg(st + GK_M), s_red);
        if (tid == 0) st[GK_AT_M] = at;
    }
    if constexpr (AFF) {
        const int32_t b = *s_bidx;
        if (b >= 0 && g >= 0)
            for (uint32_t e = __ldg(a.upd_off + g) + tid, e1 = __ldg(a.upd_off + g + 1); e < e1; e += SBD_THREADS)
                affinity_raise<false>(a, __ldg(a.upd + e), (uint32_t)b);
    }
}

// The existing pods' update entries into the zeroed counters, one warp per pod (grid-strided)
__global__ void __launch_bounds__(SBD_THREADS) k_affinity_setup(const ProfileBindArgs q) {
    const SpreadBindArgs& a = q.b;
    const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * SBD_WARPS;
    for (uint32_t e = blockIdx.x * SBD_WARPS + (threadIdx.x >> 5); e < a.E; e += warps) {
        const int32_t h = __ldg(a.ex_group + e), n = __ldg(a.ex_node + e);
        for (uint32_t i = __ldg(a.upd_off + h) + lane, i1 = __ldg(a.upd_off + h + 1); i < i1; i += 32)
            affinity_raise<true>(a, __ldg(a.upd + i), (uint32_t)n);
    }
}

// ---- ks_profile_bind and ks_node_bind: the soft scores ----


// CTA-wide minimum and maximum of one int64 pair per thread; every thread gets the result.  s holds 2 * SBD_WARPS words.
__device__ __forceinline__ void cta_minmax(int64_t& mn, int64_t& mx, int64_t* s) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        mn = min(mn, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)mn, off));
        mx = max(mx, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)mx, off));
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        s[threadIdx.x >> 5] = mn;
        s[SBD_WARPS + (threadIdx.x >> 5)] = mx;
    }
    __syncthreads();
#pragma unroll
    for (uint32_t w = 0; w < SBD_WARPS; w++) {
        mn = min(mn, s[w]);
        mx = max(mx, s[SBD_WARPS + w]);
    }
}

// The pod's soft keys: bit k when soft_skew[g * K + k] >= 1
__device__ __forceinline__ uint32_t soft_keys(const ProfileBindArgs& a, int32_t g) {
    uint32_t sk = 0;
    if (g >= 0)
        for (uint32_t k = 0; k < a.b.K; k++)
            if (__ldg(a.soft_skew + (size_t)g * a.b.K + k)) sk |= 1u << k;
    return sk;
}

// ignored (header, PodTopologySpread): the group has explicit constraints and n lacks one of its soft keys
__device__ __forceinline__ bool pts_ignored(const ProfileBindArgs& a, uint32_t sk, bool all, uint32_t n) {
    if (!all) return false;
    bool lacks = false;
#pragma unroll
    for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
        if (sk >> k & 1u) lacks |= __ldg(a.b.dom + (size_t)k * a.b.N + n) < 0;
    return lacks;
}

// The shared state of one CTA for one pod: the merged extremes, the soft weights and the domain marks
struct ProfileShared {
    int64_t key[SBD_WARPS];
    int32_t idx[SBD_WARPS];
    uint32_t ref[SBD_WARPS], aref[SBD_WARPS];
    int64_t mm[2 * SBD_WARPS];
    uint32_t bits[KS_SPREAD_MAX_KEYS * PB_SH_WORDS];
    uint32_t dom[KS_SPREAD_MAX_KEYS], lack;
    double w[KS_SPREAD_MAX_KEYS];
    int64_t imin, imax, pmin, pmax;
    uint32_t rescan;
    int32_t bidx;
};

// ks_node_bind's share of one CTA's state for one pod: per-warp refusals and raw maxima, then the grid's maxima
struct NodeShared {
    uint32_t tref[SBD_WARPS], nref[SBD_WARPS], tmax[SBD_WARPS], nmax[SBD_WARPS];
    uint32_t gtmax, gnmax;
};

// TaintToleration and NodeAffinity of a candidate from its rule word and the maxima over F (include/ksched.h, 5p)
__device__ __forceinline__ void node_parts(uint32_t rw, const NodeShared& ns, int64_t& tt, int64_t& na) {
    const int64_t t = rw >> NR_TT_SHIFT & 127u, v = rw >> NR_NA_SHIFT;
    tt = ns.gtmax == 0 ? 100 : 100 - 100 * t / ns.gtmax;
    na = ns.gnmax == 0 ? 0 : 100 * v / ns.gnmax;
}

// The row of rule words of the class of group g
__device__ __forceinline__ const uint32_t* node_row(const ProfileBindArgs& a, int32_t g) {
    return a.nrules + (size_t)__ldg(a.ncls + g + 1) * a.b.N;
}

// Pass 1: the filter; per candidate its IPA raw into iraw[], and for a group with soft keys the domains of the
// non-ignored candidates: a node-per-domain key counts its nodes, a domain below PB_SH_WORDS * 32 is marked in the CTA's
// bitmap and merged into the parity's global bitmap once per CTA, a higher one is marked there directly.  Each new
// bit counts one domain, so the partials add up to the distinct domains.  The other parity's bitmap is cleared.
// NR (ks_node_bind): the node's rule word first; the taint and node-affinity refusals and, over the candidates, the
// maxima of both raws into the CTA's partials.  FIT (ks_fit_bind, with NR): also the resource refusals, per warp in
// s_fref, into the CTA's partial pfref.  GANG (ks_gang_fit_bind) changes no code here: it gives that walk its own
// s_fref, since a function-local __shared__ array that two kernels share changes how the FIT walk addresses it.
template <int W, bool NR = false, bool FIT = false, bool GANG = false>
__device__ __forceinline__ void profile_pass1(const ProfileBindArgs& a, uint32_t p, uint32_t n0, uint32_t n1,
                                              ProfileShared& sh, NodeShared* ns = nullptr) {
    __shared__ uint32_t s_fref[SBD_WARPS]; // FIT only
    const SpreadBindArgs& b = a.b;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const BindFilter<W, true, FIT> f(a, p);
    const uint32_t sk = soft_keys(a, f.g);
    const bool all = f.g >= 0 && __ldg(a.soft_all + f.g);
    uint32_t* bits = a.bits + (size_t)(p & 1u) * a.BW;
    {
        uint32_t* other = a.bits + (size_t)(~p & 1u) * a.BW;
        for (uint32_t i = blockIdx.x * SBD_THREADS + tid; i < a.BW; i += gridDim.x * SBD_THREADS) other[i] = 0;
    }
    for (uint32_t i = tid; i < KS_SPREAD_MAX_KEYS * PB_SH_WORDS; i += SBD_THREADS) sh.bits[i] = 0;
    if (tid < KS_SPREAD_MAX_KEYS) sh.dom[tid] = 0;
    if (tid == 0) sh.lack = 0;
    uint32_t ibase[KS_SPREAD_MAX_KEYS];
#pragma unroll
    for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
        ibase[k] = f.g >= 0 && k < b.K ? __ldg(a.ibase + (size_t)f.g * b.K + k) : AFF_NONE;
    __syncthreads();
    uint32_t refused = 0, arefused = 0, lack = 0, ndom[KS_SPREAD_MAX_KEYS] = {0, 0, 0, 0};
    int64_t imin = INT64_MAX, imax = INT64_MIN;
    const uint32_t* nrow = NR ? node_row(a, f.g) : nullptr;
    uint32_t tref = 0, nref = 0, tmax = 0, nmax = 0;
    uint32_t fref = 0; // FIT only
    for (uint32_t n = n0 + tid; n < n1; n += SBD_THREADS) {
        const uint32_t rw = NR ? __ldg(nrow + n) : 0u;
        const int r = f.template test<NR>(b, n, __ldcg(b.free_cpu + n), __ldcg(b.free_mem + n), rw);
        refused += r == 1;
        arefused += r == 2;
        if constexpr (NR) {
            tref += r == 4;
            nref += r == 5;
        }
        if constexpr (FIT) fref += r == 6;
        if (r != 3) {
            a.iraw[n] = PB_NOT_CAND;
            continue;
        }
        if constexpr (NR) {
            tmax = max(tmax, rw >> NR_TT_SHIFT & 127u);
            nmax = max(nmax, rw >> NR_NA_SHIFT);
        }
        int64_t raw = 0;
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++)
            if (ibase[k] != AFF_NONE) {
                const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
                if (d >= 0) raw += __ldcg(a.icnt + ibase[k] + (uint32_t)d);
            }
        a.iraw[n] = raw;
        imin = min(imin, raw);
        imax = max(imax, raw);
        if (!sk || pts_ignored(a, sk, all, n)) continue;
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
            if (!(sk >> k & 1u)) continue;
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (d < 0) {
                lack |= 1u << k;
            } else if (a.uniq >> k & 1u) {
                ndom[k]++;
            } else if ((uint32_t)d < PB_SH_WORDS * 32) {
                atomicOr(sh.bits + k * PB_SH_WORDS + ((uint32_t)d >> 5), 1u << (d & 31));
            } else {
                uint32_t* wd = bits + a.bwo[k] + ((uint32_t)d >> 5);
                const uint32_t bit = 1u << (d & 31);
                if (!(__ldcg(wd) & bit) && !(atomicOr(wd, bit) & bit)) ndom[k]++;
            }
        }
    }
    refused = __reduce_add_sync(0xffffffffu, refused);
    arefused = __reduce_add_sync(0xffffffffu, arefused);
    lack = __reduce_or_sync(0xffffffffu, lack);
    if (lane == 0) {
        sh.ref[warp] = refused;
        sh.aref[warp] = arefused;
        if (lack) atomicOr(&sh.lack, lack);
    }
    if constexpr (NR) {
        tref = __reduce_add_sync(0xffffffffu, tref);
        nref = __reduce_add_sync(0xffffffffu, nref);
        tmax = __reduce_max_sync(0xffffffffu, tmax);
        nmax = __reduce_max_sync(0xffffffffu, nmax);
        if (lane == 0) {
            ns->tref[warp] = tref;
            ns->nref[warp] = nref;
            ns->tmax[warp] = tmax;
            ns->nmax[warp] = nmax;
        }
    }
    if constexpr (FIT) {
        fref = __reduce_add_sync(0xffffffffu, fref);
        if (lane == 0) s_fref[warp] = fref;
    }
    if (sk) {
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
            const uint32_t c = __reduce_add_sync(0xffffffffu, ndom[k]);
            if (lane == 0 && c) atomicAdd(sh.dom + k, c);
        }
    }
    cta_minmax(imin, imax, sh.mm);
    // sh.bits is complete (cta_minmax synchronises): its words into the parity's bitmap, the new bits counted
    if (sk) {
        for (uint32_t i = tid; i < KS_SPREAD_MAX_KEYS * PB_SH_WORDS; i += SBD_THREADS) {
            const uint32_t k = i / PB_SH_WORDS, v = sh.bits[i];
            if (!v) continue;
            const uint32_t old = atomicOr(bits + a.bwo[k] + i % PB_SH_WORDS, v);
            atomicAdd(sh.dom + k, (uint32_t)__popc(v & ~old));
        }
        __syncthreads();
    }
    if (tid == 0) {
        uint32_t r = 0, ar = 0;
#pragma unroll
        for (uint32_t w = 0; w < SBD_WARPS; w++) {
            r += sh.ref[w];
            ar += sh.aref[w];
        }
        b.pref[blockIdx.x] = r;
        b.paref[blockIdx.x] = ar;
        a.pimin[blockIdx.x] = imin;
        a.pimax[blockIdx.x] = imax;
        a.plack[blockIdx.x] = sh.lack;
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) a.pdom[(size_t)blockIdx.x * KS_SPREAD_MAX_KEYS + k] = sh.dom[k];
        if constexpr (NR) {
            uint32_t tr = 0, nr = 0, tm = 0, nm = 0;
#pragma unroll
            for (uint32_t w = 0; w < SBD_WARPS; w++) {
                tr += ns->tref[w];
                nr += ns->nref[w];
                tm = max(tm, ns->tmax[w]);
                nm = max(nm, ns->nmax[w]);
            }
            a.ptref[blockIdx.x] = tr;
            a.pnref[blockIdx.x] = nr;
            a.ptmax[blockIdx.x] = tm;
            a.pnmax[blockIdx.x] = nm;
        }
        if constexpr (FIT) {
            uint32_t fr = 0;
#pragma unroll
            for (uint32_t w = 0; w < SBD_WARPS; w++) fr += s_fref[w];
            a.pfref[blockIdx.x] = fr;
        }
    }
}

// Pass 2 (a pod whose group has soft keys): size_k over the grid's partials, w_k, the PodTopologySpread raw of the
// slice's candidates into praw[] (-1 when ignored) and its extremes over the non-ignored ones, max from 0
__device__ __forceinline__ void profile_pass2(const ProfileBindArgs& a, uint32_t p, uint32_t n0, uint32_t n1,
                                              ProfileShared& sh) {
    const SpreadBindArgs& b = a.b;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const int32_t g = __ldg(b.group + p);
    const uint32_t sk = soft_keys(a, g);
    const bool all = __ldg(a.soft_all + g);
    if (tid < 32) {
        uint32_t lack = 0, c[KS_SPREAD_MAX_KEYS] = {0, 0, 0, 0};
        for (uint32_t i = lane; i < gridDim.x; i += 32) {
            lack |= __ldcg(a.plack + i);
#pragma unroll
            for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) c[k] += __ldcg(a.pdom + (size_t)i * KS_SPREAD_MAX_KEYS + k);
        }
        lack = __reduce_or_sync(0xffffffffu, lack);
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
            const uint32_t size = __reduce_add_sync(0xffffffffu, c[k]) + (!all && (lack >> k & 1u));
            if (lane == 0) sh.w[k] = (sk >> k & 1u) ? __ldg(a.logw + size) : 0.0;
        }
    }
    __syncthreads();
    const uint32_t* sc = a.scnt + (size_t)g * b.S;
    int64_t mn = INT64_MAX, mx = 0;
    for (uint32_t n = n0 + tid; n < n1; n += SBD_THREADS) {
        if (a.iraw[n] == PB_NOT_CAND) continue;
        if (pts_ignored(a, sk, all, n)) {
            a.praw[n] = -1;
            continue;
        }
        double s = 0.0; // ascending k, every operation rounded on its own
#pragma unroll
        for (uint32_t k = 0; k < KS_SPREAD_MAX_KEYS; k++) {
            if (!(sk >> k & 1u)) continue;
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (d < 0) continue;
            const double t = __dadd_rn(__dmul_rn((double)__ldcg(sc + b.Pk[k] + (uint32_t)d), sh.w[k]),
                                       (double)(__ldg(a.soft_skew + (size_t)g * b.K + k) - 1u));
            s = __dadd_rn(s, t);
        }
        const int64_t raw = (int64_t)round(s); // half away from zero, as Go's math.Round
        a.praw[n] = raw;
        mn = min(mn, raw);
        mx = max(mx, raw);
    }
    cta_minmax(mn, mx, sh.mm);
    if (tid == 0) {
        a.ppmin[blockIdx.x] = mn;
        a.ppmax[blockIdx.x] = mx;
    }
}

// The normalised scores of candidate n (pts 0 for a group without soft keys)
__device__ __forceinline__ void profile_parts(const ProfileBindArgs& a, uint32_t sk, uint32_t n, const ProfileShared& sh,
                                              int64_t& pts, int64_t& ipa) {
    pts = 0;
    if (sk) {
        const int64_t r = __ldcg(a.praw + n);
        pts = r < 0 ? 0 : sh.pmax == 0 ? 100 : 100 * (sh.pmax + sh.pmin - r) / sh.pmax;
    }
    ipa = 0;
    if (sh.imax > sh.imin) {
        const int64_t r = __ldcg(a.iraw + n);
        ipa = (int64_t)__dmul_rn(100.0, __ddiv_rn((double)(r - sh.imin), (double)(sh.imax - sh.imin)));
    }
}

// Pass 3: merge the extremes, the totals of the slice's candidates and the argmax partial.  NR: also the maxima of the
// two node-rule raws, and both weighted scores in the total.
template <bool NR = false>
__device__ __forceinline__ void profile_pass3(const ProfileBindArgs& a, uint32_t p, uint32_t n0, uint32_t n1,
                                              ProfileShared& sh, NodeShared* ns = nullptr) {
    const SpreadBindArgs& b = a.b;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int32_t g = __ldg(b.group + p);
    const uint32_t sk = soft_keys(a, g);
    if (tid < 32) {
        int64_t imn = INT64_MAX, imx = INT64_MIN, pmn = INT64_MAX, pmx = 0;
        for (uint32_t i = lane; i < gridDim.x; i += 32) {
            imn = min(imn, __ldcg(a.pimin + i));
            imx = max(imx, __ldcg(a.pimax + i));
            if (sk) {
                pmn = min(pmn, __ldcg(a.ppmin + i));
                pmx = max(pmx, __ldcg(a.ppmax + i));
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            imn = min(imn, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)imn, off));
            imx = max(imx, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)imx, off));
            pmn = min(pmn, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)pmn, off));
            pmx = max(pmx, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)pmx, off));
        }
        if (lane == 0) {
            sh.imin = imn;
            sh.imax = imx;
            sh.pmin = pmn;
            sh.pmax = pmx;
        }
        if constexpr (NR) {
            uint32_t tm = 0, nm = 0;
            for (uint32_t i = lane; i < gridDim.x; i += 32) {
                tm = max(tm, __ldcg(a.ptmax + i));
                nm = max(nm, __ldcg(a.pnmax + i));
            }
            tm = __reduce_max_sync(0xffffffffu, tm);
            nm = __reduce_max_sync(0xffffffffu, nm);
            if (lane == 0) {
                ns->gtmax = tm;
                ns->gnmax = nm;
            }
        }
    }
    __syncthreads();
    const int64_t rc = __ldg(b.req_cpu + p), rm = __ldg(b.req_mem + p);
    int64_t best = INT64_MIN;
    int32_t bidx = -1;
    const uint32_t* nrow = NR ? node_row(a, g) : nullptr;
    for (uint32_t n = n0 + tid; n < n1; n += SBD_THREADS) {
        if (__ldcg(a.iraw + n) == PB_NOT_CAND) continue;
        int64_t pts, ipa;
        profile_parts(a, sk, n, sh, pts, ipa);
        int64_t key = alloc_score_rt(b.policy, __ldcg(b.free_cpu + n), __ldcg(b.free_mem + n), b.alloc_cpu,
                                     b.alloc_mem, n, rc, rm) +
                      (int64_t)a.wspread * pts + (int64_t)a.waff * ipa;
        if constexpr (NR) {
            int64_t tt, na;
            node_parts(__ldg(nrow + n), *ns, tt, na);
            key += (int64_t)a.wtaint * tt + (int64_t)a.wnaff * na;
        }
        if (key > best) { // ascending n per thread: strict '>' keeps the lowest index
            best = key;
            bidx = (int32_t)n;
        }
    }
    warp_argmax(best, bidx);
    if (lane == 0) {
        sh.key[warp] = best;
        sh.idx[warp] = bidx;
    }
    __syncthreads();
    if (warp == 0) {
        best = lane < SBD_WARPS ? sh.key[lane] : INT64_MIN;
        bidx = lane < SBD_WARPS ? sh.idx[lane] : -1;
        warp_argmax(best, bidx);
        if (lane == 0) {
            b.pkey[blockIdx.x] = best;
            b.pidx[blockIdx.x] = bidx;
        }
    }
}

// Phase B, CTA 0: spread_bind_commit's merge, binding, charge, hard counts and B/A entries (the merged key is the total,
// which key_score_rt returns unchanged for every policy this call accepts); then the parts of the winner, the soft
// counts and the bound pod's IPA entries.  The winner's parts are read from its raws and sh's extremes, which pass 3
// left in this CTA, and its policy score is the total less the weighted parts.  NR: five parts, and the first two of the
// four refusals, from the CTAs' taint and node-affinity partials.  FIT (with NR): the resource refusals in word 0 of
// five, the node-rule words after it, and free_r of the winner charged.
template <bool NR = false, bool FIT = false>
__device__ __forceinline__ void profile_commit(const ProfileBindArgs& a, uint32_t p, ProfileShared& sh,
                                               NodeShared* ns = nullptr) {
    const SpreadBindArgs& b = a.b;
    const uint32_t tid = threadIdx.x;
    spread_bind_commit<FIT ? BIND_FIT : NR ? BIND_NODE : BIND_PROFILE>(b, p, &sh.rescan, sh.ref, &sh.bidx);
    const int32_t g = __ldg(b.group + p), n = sh.bidx;
    if constexpr (FIT) {
        uint32_t fr = 0;
        if (tid < 32) {
            for (uint32_t c = threadIdx.x; c < gridDim.x; c += 32) fr += __ldcg(a.pfref + c);
            fr = __reduce_add_sync(0xffffffffu, fr);
        }
        if (tid == 0) b.out_refused[5 * (size_t)p] = fr;
        if (n >= 0 && tid < a.R)
            a.res_free[(size_t)tid * b.N + n] = __ldcg(a.res_free + (size_t)tid * b.N + n) -
                                                __ldg(a.res_req + (size_t)p * a.R + tid);
    }
    const uint32_t sk = soft_keys(a, g);
    if (tid == 0 && a.out_parts) {
        int64_t pts = 0, ipa = 0, ps = 0, tt = 0, na = 0;
        if (n >= 0) {
            profile_parts(a, sk, (uint32_t)n, sh, pts, ipa);
            ps = __ldcg(b.out_score + p) - (int64_t)a.wspread * pts - (int64_t)a.waff * ipa;
            if constexpr (NR) {
                node_parts(__ldg(node_row(a, g) + n), *ns, tt, na);
                ps -= (int64_t)a.wtaint * tt + (int64_t)a.wnaff * na;
            }
        }
        constexpr size_t PW = bind_part_words(FIT ? BIND_FIT : NR ? BIND_NODE : BIND_PROFILE);
        a.out_parts[PW * p] = ps;
        a.out_parts[PW * p + 1] = pts;
        a.out_parts[PW * p + 2] = ipa;
        if constexpr (NR) {
            a.out_parts[PW * p + 3] = tt;
            a.out_parts[PW * p + 4] = na;
        }
    }
    if constexpr (NR) {
        uint32_t tr = 0, nr = 0;
        if (tid < 32) { // the CTAs' partials across the warp, as spread_bind_commit merges its own
            for (uint32_t c = threadIdx.x; c < gridDim.x; c += 32) {
                tr += __ldcg(a.ptref + c);
                nr += __ldcg(a.pnref + c);
            }
            tr = __reduce_add_sync(0xffffffffu, tr);
            nr = __reduce_add_sync(0xffffffffu, nr);
        }
        if (tid == 0) {
            if constexpr (FIT) { // after the resource word
                b.out_refused[5 * (size_t)p + 1] = tr;
                b.out_refused[5 * (size_t)p + 2] = nr;
            } else {
                b.out_refused[4 * (size_t)p] = tr;
                b.out_refused[4 * (size_t)p + 1] = nr;
            }
        }
    }
    if (n < 0 || g < 0) return;
    if (tid == 0 && sk && !pts_ignored(a, sk, __ldg(a.soft_all + g), (uint32_t)n)) {
        uint32_t* sc = a.scnt + (size_t)g * b.S;
        for (uint32_t k = 0; k < b.K; k++) {
            if (!(sk >> k & 1u)) continue;
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (d >= 0) sc[b.Pk[k] + (uint32_t)d] = __ldcg(sc + b.Pk[k] + (uint32_t)d) + 1;
        }
    }
    // entries of one list name distinct (group, key) arrays: no atomics
    for (uint32_t e = __ldg(a.iupd_off + g) + tid, e1 = __ldg(a.iupd_off + g + 1); e < e1; e += SBD_THREADS) {
        const uint32_t en = __ldg(a.iupd + e), h = en & 0xffffu, k = en >> 16;
        const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
        if (d < 0) continue;
        int64_t* c = a.icnt + __ldg(a.ibase + (size_t)h * b.K + k) + (uint32_t)d;
        *c = __ldcg(c) + __ldg(a.icoef + e);
    }
}

// The existing pods' IPA entries into the zeroed counters, one warp per pod (grid-strided)
__global__ void __launch_bounds__(SBD_THREADS) k_profile_setup(const ProfileBindArgs a) {
    const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * SBD_WARPS;
    for (uint32_t e = blockIdx.x * SBD_WARPS + (threadIdx.x >> 5); e < a.b.E; e += warps) {
        const int32_t h = __ldg(a.b.ex_group + e), n = __ldg(a.b.ex_node + e);
        for (uint32_t i = __ldg(a.iupd_off + h) + lane, i1 = __ldg(a.iupd_off + h + 1); i < i1; i += 32) {
            const uint32_t en = __ldg(a.iupd + i), g = en & 0xffffu, k = en >> 16;
            const int32_t d = __ldg(a.b.dom + (size_t)k * a.b.N + n);
            if (d < 0) continue;
            atomicAdd(reinterpret_cast<unsigned long long*>(a.icnt + __ldg(a.ibase + (size_t)g * a.b.K + k) + (uint32_t)d),
                      (unsigned long long)(int64_t)__ldg(a.icoef + i));
        }
    }
}

// ---- ks_gang_fit_bind: the rollback of a gang (include/ksched.h, 5s) ----

// CTA 0, after the commit of the gang's last pod: its pods [q0, q1) that bound are unbound and every piece of state their
// commits changed goes back to its value before the gang.  The additive state is reversed by subtraction, per bound pod,
// with the same node, update entries and soft-count condition that raised it; the sums wrap in two's complement, so the
// order does not matter and atomics may run the pods in parallel.  Each group the gang charged (stamp = gang + 1 marks
// it once) then gets its gk words from the restored counts, as k_bind_setup forms them: m = the minimum over the
// eligible domains and the domains at m, except under minDomains (FORCED) or with no eligible domain, which no commit
// changes.  Each group h whose any-flag a bound pod raised gets the flag from its restored A counters: the flag is 1
// exactly when some pod of M_h counts in one of them.  Refusal words stay as the pods' turns wrote them.
__device__ __forceinline__ void gang_rollback(const ProfileBindArgs& a, uint32_t q0, uint32_t q1, uint32_t stamp,
                                           uint32_t* s_red) {
    __shared__ uint32_t s_n[2]; // groups listed: for their gk words, for their any-flag
    const SpreadBindArgs& b = a.b;
    const uint32_t tid = threadIdx.x;
    if (tid < 2) s_n[tid] = 0;
    __syncthreads(); // also orders the commit's writes before the reads below
    for (uint32_t q = q0 + tid; q < q1; q += SBD_THREADS) {
        const int32_t n = __ldcg(b.out_idx + q);
        if (n < 0) continue;
        b.out_idx[q] = -1;
        b.out_score[q] = 0;
        if (a.out_parts)
            for (uint32_t i = 0; i < 5; i++) a.out_parts[5 * (size_t)q + i] = 0;
        atomicAdd(reinterpret_cast<unsigned long long*>(b.free_cpu + n), (unsigned long long)__ldg(b.req_cpu + q));
        atomicAdd(reinterpret_cast<unsigned long long*>(b.free_mem + n), (unsigned long long)__ldg(b.req_mem + q));
        for (uint32_t r = 0; r < a.R; r++)
            atomicAdd(reinterpret_cast<unsigned long long*>(a.res_free + (size_t)r * b.N + n),
                      (unsigned long long)__ldg(a.res_req + (size_t)q * a.R + r));
        const int32_t g = __ldg(b.group + q);
        if (g < 0) continue;
        const uint32_t ck = constrained_keys(b, g), sk = soft_keys(a, g);
        const bool soft = sk && !pts_ignored(a, sk, __ldg(a.soft_all + g), (uint32_t)n);
        for (uint32_t k = 0; k < b.K; k++) {
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (ck >> k & 1u) atomicSub(b.cnt + (size_t)g * b.S + b.Pk[k] + (uint32_t)d, 1u);
            if (soft && (sk >> k & 1u) && d >= 0) atomicSub(a.scnt + (size_t)g * b.S + b.Pk[k] + (uint32_t)d, 1u);
        }
        if (ck && atomicExch(a.gmark + g, stamp) != stamp) a.glist[atomicAdd(s_n, 1u)] = (uint32_t)g;
        for (uint32_t e = __ldg(b.upd_off + g), e1 = __ldg(b.upd_off + g + 1); e < e1; e++) {
            const uint32_t en = __ldg(b.upd + e), h = en & 0xffffu, k = en >> 16 & 0xfu, kind = en >> 20;
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (d < 0) continue;
            atomicSub(b.acnt + __ldg(b.abase + ((size_t)h * b.K + k) * 2 + kind) + (uint32_t)d, 1u);
            if (kind && atomicExch(a.gmark + b.G + h, stamp) != stamp) a.glist[b.G + atomicAdd(s_n + 1, 1u)] = h;
        }
        for (uint32_t e = __ldg(a.iupd_off + g), e1 = __ldg(a.iupd_off + g + 1); e < e1; e++) {
            const uint32_t en = __ldg(a.iupd + e), h = en & 0xffffu, k = en >> 16;
            const int32_t d = __ldg(b.dom + (size_t)k * b.N + n);
            if (d < 0) continue;
            atomicAdd(reinterpret_cast<unsigned long long*>(a.icnt + __ldg(a.ibase + (size_t)h * b.K + k) + (uint32_t)d),
                      (unsigned long long)-(int64_t)__ldg(a.icoef + e));
        }
    }
    __syncthreads();
    for (uint32_t i = 0, n_gk = s_n[0]; i < n_gk; i++) {
        const uint32_t g = __ldcg(a.glist + i), ck = constrained_keys(b, (int32_t)g);
        for (uint32_t k = 0; k < b.K; k++) {
            uint32_t* st = b.gk + ((size_t)g * b.K + k) * GK_WORDS;
            if (!(ck >> k & 1u) || (__ldcg(st + GK_FLAGS) & GK_FORCED) || __ldcg(st + GK_NE) == 0) continue;
            const size_t base = (size_t)g * b.S + b.Pk[k];
            uint32_t mn = 0xffffffffu;
            for (uint32_t d = tid; d < b.Dk[k]; d += SBD_THREADS)
                if (b.elig[base + d]) mn = min(mn, __ldcg(b.cnt + base + d));
            mn = cta_min(mn, s_red);
            const uint32_t at = domains_at(b, g, k, mn, s_red);
            if (tid == 0) {
                st[GK_M] = mn;
                st[GK_AT_M] = at;
            }
        }
    }
    for (uint32_t i = 0, n_any = s_n[1]; i < n_any; i++) {
        const uint32_t h = __ldcg(a.glist + b.G + i);
        uint32_t any = 0;
        for (uint32_t k = 0; k < b.K; k++) {
            const uint32_t base = __ldg(b.abase + ((size_t)h * b.K + k) * 2 + 1);
            if (base == AFF_NONE) continue;
            for (uint32_t d = tid; d < b.Dk[k]; d += SBD_THREADS) any |= __ldcg(b.acnt + base + d);
        }
        any = __syncthreads_or(any != 0);
        if (tid == 0) b.acnt[b.any_base + h] = any ? 1u : 0u;
    }
}

// ks_node_bind: one rule word per (class c, node n) over the grid-strided C x N pairs (include/ksched.h, 5p)
__global__ void __launch_bounds__(SBD_THREADS) k_node_rules_setup(const ProfileBindArgs a) {
    const uint64_t total = (uint64_t)a.C * a.b.N;
    for (uint64_t i = (uint64_t)blockIdx.x * SBD_THREADS + threadIdx.x; i < total; i += (uint64_t)gridDim.x * SBD_THREADS) {
        const uint32_t c = (uint32_t)(i / a.b.N), n = (uint32_t)(i % a.b.N);
        const uint64_t hard = __ldg(a.taint_hard + n) & ~__ldg(a.ctol + 2 * c);
        const uint32_t tt = __popcll(__ldg(a.taint_soft + n) & ~__ldg(a.ctol + 2 * c + 1));
        bool has_req = false, req_ok = false;
        uint32_t na = 0;
        for (uint32_t t = __ldg(a.cterm_off + c), t1 = __ldg(a.cterm_off + c + 1); t < t1; t++) {
            const uint32_t x0 = __ldg(a.cexpr_off + t), x1 = __ldg(a.cexpr_off + t + 1);
            bool ok = x1 > x0; // a term with no expression matches nothing
            for (uint32_t x = x0; x < x1 && ok; x++) {
                const uint32_t k = __ldg(a.cexpr_key + x);
                const int32_t d = __ldg(a.ndom + (size_t)k * a.b.N + n);
                const uint32_t bit = d < 0 ? a.NDk[k] : (uint32_t)d;
                ok = __ldg(a.nset + __ldg(a.cexpr_set + x) + bit / 64) >> (bit % 64) & 1u;
            }
            const uint32_t w = __ldg(a.cterm_w + t);
            if (w == 0) {
                has_req = true;
                req_ok |= ok;
            } else if (ok) {
                na += w;
            }
        }
        const bool aff_ok = !has_req || req_ok;
        const uint32_t reason = hard ? NR_TAINT : aff_ok ? 0u : NR_AFFINITY;
        a.nrules[i] = reason | (aff_ok ? NR_AFF_OK : 0u) | tt << NR_TT_SHIFT | na << NR_NA_SHIFT;
    }
}

// The walk of every bind call: one cooperative launch, one node slice per CTA, the pods in queue order with grid
// barriers between their phases.  SPREAD and AFFINITY run phase A and phase B; PROFILE and NODE run pass 1, pass 2 when
// the pod's group has soft keys, pass 3 and the commit.  GANG_FIT is FIT, and after the commit of a gang's last pod CTA 0
// writes the gang's count and rolls it back when it is short, before that pod's last barrier.  Each family declares only
// its own shared state.
template <int W, BindMode M>
__global__ void __launch_bounds__(SBD_THREADS, 1) k_bind_seq(const ProfileBindArgs a) {
    constexpr bool AFF = M != BIND_SPREAD, GANG = M == BIND_GANG_FIT, FIT = M == BIND_FIT || GANG,
                   NR = M == BIND_NODE || FIT;
    cg::grid_group grid = cg::this_grid();
    const uint32_t G = gridDim.x;
    const uint32_t chunk = (a.b.N + G - 1) / G, n0 = min(a.b.N, blockIdx.x * chunk), n1 = min(a.b.N, n0 + chunk);
    if constexpr (M == BIND_SPREAD || M == BIND_AFFINITY) {
        __shared__ int64_t s_key[SBD_WARPS];
        __shared__ int32_t s_idx[SBD_WARPS];
        __shared__ uint32_t s_ref[SBD_WARPS], s_aref[SBD_WARPS]; // s_aref: AFF only
        __shared__ uint32_t s_rescan;
        __shared__ int32_t s_bidx; // AFF only
        for (uint32_t p = 0; p < a.b.P; p++) {
            spread_bind_scan<W, AFF>(a.b, p, n0, n1, s_key, s_idx, s_ref, s_aref);
            __threadfence();
            grid.sync();
            if (blockIdx.x == 0) spread_bind_commit<M>(a.b, p, &s_rescan, s_ref, &s_bidx);
            __threadfence();
            grid.sync();
        }
    } else {
        __shared__ ProfileShared sh;
        __shared__ NodeShared ns; // NR only
        uint32_t j = 0, placed = 0; // GANG, CTA 0: the current gang and its pods bound so far
        for (uint32_t p = 0; p < a.b.P; p++) {
            profile_pass1<W, NR, FIT, GANG>(a, p, n0, n1, sh, &ns);
            __threadfence();
            grid.sync();
            if (soft_keys(a, __ldg(a.b.group + p))) { // uniform: every CTA knows the pod's group
                profile_pass2(a, p, n0, n1, sh);
                __threadfence();
            grid.sync();
            }
            profile_pass3<NR>(a, p, n0, n1, sh, &ns);
            __threadfence();
            grid.sync();
            if (blockIdx.x == 0) {
                profile_commit<NR, FIT>(a, p, sh, &ns);
                if constexpr (GANG) { // after the gang's last pod: its count, and the rollback before the barrier
                    placed += sh.bidx >= 0;
                    if (p + 1 == __ldg(a.goff + j + 1)) {
                        if (threadIdx.x == 0) a.gplaced[j] = placed;
                        if (placed < __ldg(a.gmin + j)) gang_rollback(a, __ldg(a.goff + j), p + 1, j + 1, sh.ref);
                        j++;
                        placed = 0;
                    }
                }
            }
            __threadfence();
            grid.sync();
        }
    }
}

cudaError_t launch_node_rules(const ProfileBindArgs& a, cudaStream_t st) {
    k_node_rules_setup<<<a.rules_grid, SBD_THREADS, 0, st>>>(a);
    g_launches++;
    return cudaGetLastError();
}

uint32_t bind_setup_grid(uint32_t G, int sms) { return std::max(1u, std::min<uint32_t>(G, 4u * (uint32_t)sms)); }

cudaError_t launch_bind(BindMode mode, const ProfileBindArgs& a, uint64_t acnt_words, uint32_t W, cudaStream_t st) {
    return with_label_width(W, [&](auto w) {
        constexpr int LW = decltype(w)::value;
        const SpreadBindArgs& b = a.b;
        const bool gang = mode == BIND_GANG_FIT, fit = mode == BIND_FIT || gang, nr = mode == BIND_NODE || fit,
                   soft = mode == BIND_PROFILE || nr;
        const auto launched = [](uint32_t n) {
            g_launches += n;
            return cudaGetLastError();
        };
        cudaError_t e;
        if (nr && (e = launch_node_rules(a, st)) != cudaSuccess) return e;
        if (b.G) {
            if (nr) k_bind_setup<LW, true><<<b.setup_grid, SBD_THREADS, 0, st>>>(a);
            else k_bind_setup<LW, false><<<b.setup_grid, SBD_THREADS, 0, st>>>(a);
            if ((e = launched(1)) != cudaSuccess) return e;
        }
        if (mode != BIND_SPREAD) {
            e = cudaMemsetAsync(b.acnt, 0, acnt_words * 4, st);
            if (soft) {
                if (e == cudaSuccess) e = cudaMemsetAsync(a.icnt, 0, a.iwords * 8, st);
                if (e == cudaSuccess) e = cudaMemsetAsync(a.bits, 0, (size_t)a.BW * 8, st);
                if (e == cudaSuccess && b.G && b.S)
                    e = b.existing
                            ? cudaMemcpyAsync(a.scnt, b.existing, (size_t)b.G * b.S * 4, cudaMemcpyDeviceToDevice, st)
                            : cudaMemsetAsync(a.scnt, 0, (size_t)b.G * b.S * 4, st);
                if (e == cudaSuccess && fit && a.R)
                    e = cudaMemcpyAsync(a.res_free, a.res_node_free, (size_t)a.R * b.N * 8, cudaMemcpyDeviceToDevice, st);
                if (e == cudaSuccess && gang && b.G) e = cudaMemsetAsync(a.gmark, 0, (size_t)b.G * 8, st);
            }
            if (e != cudaSuccess) return e;
            if (b.E) {
                k_affinity_setup<<<b.aff_grid, SBD_THREADS, 0, st>>>(a);
                if (soft) k_profile_setup<<<b.aff_grid, SBD_THREADS, 0, st>>>(a);
                if ((e = launched(soft ? 2 : 1)) != cudaSuccess) return e;
            }
        }
        const void* walk = mode == BIND_SPREAD     ? reinterpret_cast<const void*>(k_bind_seq<LW, BIND_SPREAD>)
                           : mode == BIND_AFFINITY ? reinterpret_cast<const void*>(k_bind_seq<LW, BIND_AFFINITY>)
                           : mode == BIND_PROFILE  ? reinterpret_cast<const void*>(k_bind_seq<LW, BIND_PROFILE>)
                           : mode == BIND_NODE     ? reinterpret_cast<const void*>(k_bind_seq<LW, BIND_NODE>)
                           : mode == BIND_FIT      ? reinterpret_cast<const void*>(k_bind_seq<LW, BIND_FIT>)
                                                   : reinterpret_cast<const void*>(k_bind_seq<LW, BIND_GANG_FIT>);
        ProfileBindArgs c = a;
        void* args[] = {&c};
        e = cudaLaunchCooperativeKernel(walk, dim3(b.grid), dim3(SBD_THREADS), args, 0, st);
        if (e == cudaSuccess) g_launches++;
        return e;
    });
}

} // namespace ks
