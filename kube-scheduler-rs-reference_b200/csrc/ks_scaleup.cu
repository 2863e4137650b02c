// ks_scaleup.cu — scale-up estimate (ks_scaleup_estimate, include/ksched.h; DESIGN.md 5g), sm_90a.
// Templates are independent, so each one is a CTA of k_scaleup_pack: it compacts its eligible pods in pod order, sorts
// them by the order key with ks_sort.cuh's stable LSD radix sort in its own scratch slot, and then one warp walks them
// through the first-fit packing with the open nodes' remaining capacity in shared memory.  k_scaleup_reasons counts the
// per-pod rejection reasons over the templates without atomics, one thread per pod.  k_fit_scaleup_pack and
// k_fit_scaleup_reasons are the same two passes under ks_fit_bind's full filter (ks_fit_scaleup_estimate, DESIGN.md 5v).
#include "ks_launch.h"
#include "ks_sort.cuh"

namespace ks {

constexpr int SU_THREADS = 256; // 8 warps; the radix pass gives each thread one of the 256 digits
constexpr int SU_CHUNK = 256; // templates staged in shared memory per step of k_scaleup_reasons
static_assert(SU_THREADS == SORT_THREADS, "one thread per radix digit");

// The order key of a pod for a template: req_cpu * A_m + req_mem * A_c.  Requests lie in [0, 2^36] / [0, 2^55] and
// allocatables in [1, 2^26] / [1, 2^45] (checked on the host), so the key fits 128 bits; for an eligible pod (req <= F
// <= A) it is below 2^73.
__device__ __forceinline__ unsigned __int128 su_key(int64_t rc, int64_t rm, int64_t ac, int64_t am) {
    return (unsigned __int128)(uint64_t)rc * (uint64_t)am + (unsigned __int128)(uint64_t)rm * (uint64_t)ac;
}

// Digit of the pod's key at `shift`, inverted so that an ascending stable sort orders the keys descending and keeps
// equal keys in pod order.
__device__ __forceinline__ uint32_t su_digit(const PodView& pv, uint32_t p, int64_t ac, int64_t am, uint32_t shift) {
    const unsigned __int128 k = su_key(__ldg(pv.req_cpu + p), __ldg(pv.req_mem + p), ac, am);
    return 255u - ((uint32_t)(k >> shift) & 255u);
}

struct SuShared {
    int64_t rem_cpu[KS_SCALEUP_MAX_NODES]; // remaining capacity of the open nodes, by ordinal
    int64_t rem_mem[KS_SCALEUP_MAX_NODES];
    SortShared sort; // the radix passes and the block scan
};

template <int W>
__global__ void __launch_bounds__(SU_THREADS) k_scaleup_pack(PodView pv, ScaleupArgs a) {
    __shared__ SuShared s;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t P = pv.P;
    uint32_t* const buf0 = a.scratch + (uint64_t)blockIdx.x * 2 * P;
    uint32_t* const buf1 = buf0 + P;
    for (uint32_t t = blockIdx.x; t < a.T; t += gridDim.x) {
        __syncthreads(); // the previous template's walk is done with the scratch slot and the open nodes
        const int64_t ac = a.alloc_cpu[t], am = a.alloc_mem[t], fc = a.free_cpu[t], fm = a.free_mem[t];
        uint64_t lab[W];
#pragma unroll
        for (int w = 0; w < W; w++) lab[w] = a.labels[(uint64_t)t * W + w];
        // 1. eligible pods, compacted in pod order
        uint32_t E = 0;
        for (uint32_t b = 0; b < P; b += SU_THREADS) {
            const uint32_t p = b + threadIdx.x;
            bool ok = false;
            if (p < P) {
                ok = (pv.req_cpu[p] <= fc) & (pv.req_mem[p] <= fm);
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= pv.sel[(uint64_t)p * W + w] & ~lab[w];
                ok &= miss == 0;
            }
            uint32_t total;
            const uint32_t pre = cta_block_scan(ok ? 1u : 0u, s.sort.wsum, total);
            if (ok) buf0[E + pre] = p;
            E += total;
        }
        __syncthreads();
        // 2. stable sort by the key, descending, over the digits the largest possible key has (fc, fm >= 0 when E > 0)
        uint32_t* src = buf0;
        uint32_t* dst = buf1;
        if (E > 1) {
            const unsigned __int128 kmax = su_key(fc, fm, ac, am);
            const uint64_t hi = (uint64_t)(kmax >> 64), lo = (uint64_t)kmax;
            const uint32_t bits = hi ? 128u - __clzll(hi) : lo ? 64u - __clzll(lo) : 0u;
            for (uint32_t shift = 0; shift < bits; shift += 8) {
                cta_radix_pass(src, dst, E, [&](uint32_t p) { return su_digit(pv, p, ac, am, shift); }, s.sort);
                uint32_t* x = src;
                src = dst;
                dst = x;
            }
        }
        // 3. first fit, one warp: 32 pods prefetched per step, the open nodes scanned 32 ordinals per ballot
        if (warp != 0) continue;
        const uint32_t maxn = a.max_nodes[t];
        uint32_t nodes = 0, placed = 0;
        int64_t used_cpu = 0, used_mem = 0;
        for (uint32_t b = 0; b < E; b += 32) {
            const uint32_t k = b + lane;
            const uint32_t kp = k < E ? src[k] : 0u;
            const int64_t kc = k < E ? pv.req_cpu[kp] : 0, km = k < E ? pv.req_mem[kp] : 0;
            const uint32_t cnt = min(32u, E - b);
            for (uint32_t j = 0; j < cnt; j++) {
                const uint32_t p = __shfl_sync(0xffffffffu, kp, j);
                const int64_t c = __shfl_sync(0xffffffffu, kc, j), m = __shfl_sync(0xffffffffu, km, j);
                int32_t node = -1;
                for (uint32_t o0 = 0; o0 < nodes; o0 += 32) {
                    const uint32_t o = o0 + lane;
                    const uint32_t fit = __ballot_sync(0xffffffffu, o < nodes && c <= s.rem_cpu[o] && m <= s.rem_mem[o]);
                    if (fit) {
                        node = (int32_t)(o0 + __ffs(fit) - 1);
                        break;
                    }
                }
                if (node < 0 && nodes < maxn) {
                    node = (int32_t)nodes++;
                    if (lane == 0) {
                        s.rem_cpu[node] = fc;
                        s.rem_mem[node] = fm;
                    }
                }
                if (node >= 0) {
                    if (lane == 0) {
                        s.rem_cpu[node] -= c;
                        s.rem_mem[node] -= m;
                        if (a.out_node) a.out_node[(uint64_t)t * P + p] = node;
                    }
                    placed++;
                    used_cpu += c;
                    used_mem += m;
                }
                __syncwarp(); // lane 0's update is seen by the next pod's scan
            }
        }
        if (lane == 0) {
            ks_scaleup_option r;
            r.nodes = nodes;
            r.placed = placed;
            r.eligible = E;
            r.utilization = 0;
            if (nodes) {
                const int64_t pc = used_cpu * 100 / ((int64_t)nodes * ac), pm = used_mem * 100 / ((int64_t)nodes * am);
                r.utilization = (int32_t)((pc + pm) / 2);
            }
            r.used_cpu = used_cpu;
            r.used_mem = used_mem;
            a.rows[t] = r;
        }
    }
}

// One thread per pod: ks_explain's four counts over the templates (capacity F as the free values), staged SU_CHUNK
// templates at a time.
template <int W>
__global__ void __launch_bounds__(SU_THREADS) k_scaleup_reasons(PodView pv, ScaleupArgs a) {
    __shared__ int64_t s_fc[SU_CHUNK], s_fm[SU_CHUNK];
    __shared__ uint64_t s_lab[W][SU_CHUNK];
    const uint32_t p = blockIdx.x * SU_THREADS + threadIdx.x;
    const bool live = p < pv.P;
    const int64_t rc = live ? pv.req_cpu[p] : 0, rm = live ? pv.req_mem[p] : 0;
    uint64_t sel[W];
#pragma unroll
    for (int w = 0; w < W; w++) sel[w] = live ? pv.sel[(uint64_t)p * W + w] : 0;
    uint32_t cpu = 0, mem = 0, nores = 0, nosel = 0;
    for (uint32_t t0 = 0; t0 < a.T; t0 += SU_CHUNK) {
        const uint32_t n = min((uint32_t)SU_CHUNK, a.T - t0);
        __syncthreads();
        if (threadIdx.x < n) {
            const uint32_t t = t0 + threadIdx.x;
            s_fc[threadIdx.x] = a.free_cpu[t];
            s_fm[threadIdx.x] = a.free_mem[t];
#pragma unroll
            for (int w = 0; w < W; w++) s_lab[w][threadIdx.x] = a.labels[(uint64_t)t * W + w];
        }
        __syncthreads();
        for (uint32_t j = 0; j < n; j++) {
            const bool fc = rc > s_fc[j], fm = rm > s_fm[j];
            uint64_t miss = 0;
#pragma unroll
            for (int w = 0; w < W; w++) miss |= sel[w] & ~s_lab[w][j];
            cpu += fc;
            mem += fm;
            nores += fc | fm;
            nosel += !(fc | fm) && miss != 0;
        }
    }
    if (live) reinterpret_cast<uint4*>(a.reasons)[p] = make_uint4(cpu, mem, nores, nosel);
}

// ---- under the full filter (ks_fit_scaleup_estimate, DESIGN.md 5v) ----
constexpr uint32_t FSU_RMASK = (1u << KS_BIND_MAX_RESOURCES) - 1u;

// Pod p's refusal stage on an empty node of template t, in ks_fit_bind's filter order: 0 cpu, memory or selector, 1 a
// resource, 2 an untolerated hard taint, 3 required node affinity, 4 eligible.  nf(r) = node_free of r at t; q[r] the
// pod's requests, rmask the non-zero ones (upstream's zero skip); rw the rule word of (class(group[p]), t).
template <int W, class NF>
__device__ __forceinline__ uint32_t fsu_stage(int64_t rc, int64_t rm, const uint64_t (&sel)[W], int64_t fc, int64_t fm,
                                              const uint64_t (&lab)[W], const int64_t (&q)[KS_BIND_MAX_RESOURCES],
                                              uint32_t rmask, NF nf, uint32_t rw) {
    uint64_t miss = 0;
#pragma unroll
    for (int w = 0; w < W; w++) miss |= sel[w] & ~lab[w];
    if (rc > fc || rm > fm || miss != 0) return 0;
    bool fit_r = true;
#pragma unroll
    for (int r = 0; r < (int)KS_BIND_MAX_RESOURCES; r++)
        if (rmask >> r & 1u) fit_r &= q[r] <= nf(r);
    if (!fit_r) return 1;
    const uint32_t reason = rw & NR_REASON;
    return reason == NR_TAINT ? 2u : reason == NR_AFFINITY ? 3u : 4u;
}

// k_scaleup_pack with the full filter: the compaction also needs the class's rule word at t to pass and every requested
// resource to fit node_free; the walk keeps 2 + R remainders per open ordinal in dynamic shared memory, column d of
// ordinal o at d * KS_SCALEUP_MAX_NODES + o (cpu, memory, then the R resources), and a lane's ordinal fits when cpu,
// memory and each resource in the pod's request mask fit.  Placing a pod subtracts every request.
template <int W>
__global__ void __launch_bounds__(SU_THREADS) k_fit_scaleup_pack(PodView pv, ScaleupArgs a, FitScaleupArgs f) {
    extern __shared__ int64_t fsu_rem[]; // [(2 + R) * KS_SCALEUP_MAX_NODES]
    __shared__ SortShared sort;
    __shared__ int64_t s_nf[KS_BIND_MAX_RESOURCES];
    __shared__ int64_t s_req[32][KS_BIND_MAX_RESOURCES]; // the walk's 32 prefetched pods' requests
    __shared__ int64_t s_used[KS_BIND_MAX_RESOURCES];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t P = pv.P, R = f.R, T = a.T;
    uint32_t* const buf0 = a.scratch + (uint64_t)blockIdx.x * 2 * P;
    uint32_t* const buf1 = buf0 + P;
    for (uint32_t t = blockIdx.x; t < T; t += gridDim.x) {
        __syncthreads(); // the previous template's walk is done with the scratch slot, the open nodes and s_nf
        const int64_t ac = a.alloc_cpu[t], am = a.alloc_mem[t], fc = a.free_cpu[t], fm = a.free_mem[t];
        uint64_t lab[W];
#pragma unroll
        for (int w = 0; w < W; w++) lab[w] = a.labels[(uint64_t)t * W + w];
        if (threadIdx.x < R) s_nf[threadIdx.x] = f.node_free[(uint64_t)threadIdx.x * T + t];
        __syncthreads();
        // 1. eligible pods, compacted in pod order
        uint32_t E = 0;
        for (uint32_t b = 0; b < P; b += SU_THREADS) {
            const uint32_t p = b + threadIdx.x;
            bool ok = false;
            if (p < P) {
                uint64_t sel[W];
#pragma unroll
                for (int w = 0; w < W; w++) sel[w] = pv.sel[(uint64_t)p * W + w];
                int64_t q[KS_BIND_MAX_RESOURCES];
                uint32_t rmask = 0;
#pragma unroll
                for (int r = 0; r < (int)KS_BIND_MAX_RESOURCES; r++) {
                    q[r] = r < (int)R ? f.req[(uint64_t)p * R + r] : 0;
                    rmask |= (q[r] != 0 ? 1u : 0u) << r;
                }
                const uint32_t rw = __ldg(f.nrules + (uint64_t)__ldg(f.ncls + f.group[p] + 1) * T + t);
                ok = fsu_stage<W>(pv.req_cpu[p], pv.req_mem[p], sel, fc, fm, lab, q, rmask,
                                  [&](int r) { return s_nf[r]; }, rw) == 4u;
            }
            uint32_t total;
            const uint32_t pre = cta_block_scan(ok ? 1u : 0u, sort.wsum, total);
            if (ok) buf0[E + pre] = p;
            E += total;
        }
        __syncthreads();
        // 2. k_scaleup_pack's sort
        uint32_t* src = buf0;
        uint32_t* dst = buf1;
        if (E > 1) {
            const unsigned __int128 kmax = su_key(fc, fm, ac, am);
            const uint64_t hi = (uint64_t)(kmax >> 64), lo = (uint64_t)kmax;
            const uint32_t bits = hi ? 128u - __clzll(hi) : lo ? 64u - __clzll(lo) : 0u;
            for (uint32_t shift = 0; shift < bits; shift += 8) {
                cta_radix_pass(src, dst, E, [&](uint32_t p) { return su_digit(pv, p, ac, am, shift); }, sort);
                uint32_t* x = src;
                src = dst;
                dst = x;
            }
        }
        // 3. first fit, one warp: 32 pods prefetched per step (their R requests in shared memory), 32 ordinals per
        // ballot
        if (warp != 0) continue;
        int64_t* const rem_c = fsu_rem;
        int64_t* const rem_m = fsu_rem + KS_SCALEUP_MAX_NODES;
        int64_t* const rem_r = fsu_rem + 2 * KS_SCALEUP_MAX_NODES; // resource r at r * KS_SCALEUP_MAX_NODES
        const uint32_t maxn = a.max_nodes[t];
        uint32_t nodes = 0, placed = 0;
        int64_t used_cpu = 0, used_mem = 0;
        if (lane < KS_BIND_MAX_RESOURCES) s_used[lane] = 0;
        for (uint32_t b = 0; b < E; b += 32) {
            const uint32_t k = b + lane;
            const uint32_t kp = k < E ? src[k] : 0u;
            const int64_t kc = k < E ? pv.req_cpu[kp] : 0, km = k < E ? pv.req_mem[kp] : 0;
            uint32_t kmask = 0;
            for (uint32_t r = 0; r < R; r++) {
                const int64_t q = k < E ? f.req[(uint64_t)kp * R + r] : 0;
                s_req[lane][r] = q;
                kmask |= (q != 0 ? 1u : 0u) << r;
            }
            __syncwarp();
            const uint32_t cnt = min(32u, E - b);
            for (uint32_t j = 0; j < cnt; j++) {
                const uint32_t p = __shfl_sync(0xffffffffu, kp, j), rmask = __shfl_sync(0xffffffffu, kmask, j);
                const int64_t c = __shfl_sync(0xffffffffu, kc, j), m = __shfl_sync(0xffffffffu, km, j);
                int32_t node = -1;
                for (uint32_t o0 = 0; o0 < nodes; o0 += 32) {
                    const uint32_t o = o0 + lane;
                    bool ok = o < nodes && c <= rem_c[o] && m <= rem_m[o];
#pragma unroll
                    for (int r = 0; r < (int)KS_BIND_MAX_RESOURCES; r++) // rmask is warp-uniform
                        if (rmask >> r & 1u) ok &= o < nodes && s_req[j][r] <= rem_r[r * KS_SCALEUP_MAX_NODES + o];
                    const uint32_t fit = __ballot_sync(0xffffffffu, ok);
                    if (fit) {
                        node = (int32_t)(o0 + __ffs(fit) - 1);
                        break;
                    }
                }
                if (node < 0 && nodes < maxn) {
                    node = (int32_t)nodes++;
                    if (lane == 0) {
                        rem_c[node] = fc;
                        rem_m[node] = fm;
                        for (uint32_t r = 0; r < R; r++) rem_r[r * KS_SCALEUP_MAX_NODES + node] = s_nf[r];
                    }
                }
                if (node >= 0) {
                    if (lane == 0) {
                        rem_c[node] -= c;
                        rem_m[node] -= m;
                        for (uint32_t r = 0; r < R; r++) {
                            rem_r[r * KS_SCALEUP_MAX_NODES + node] -= s_req[j][r];
                            s_used[r] += s_req[j][r];
                        }
                        if (a.out_node) a.out_node[(uint64_t)t * P + p] = node;
                    }
                    placed++;
                    used_cpu += c;
                    used_mem += m;
                }
                __syncwarp(); // lane 0's update is seen by the next pod's scan
            }
        }
        if (lane == 0) {
            ks_scaleup_option r;
            r.nodes = nodes;
            r.placed = placed;
            r.eligible = E;
            r.utilization = 0;
            if (nodes) {
                const int64_t pc = used_cpu * 100 / ((int64_t)nodes * ac), pm = used_mem * 100 / ((int64_t)nodes * am);
                r.utilization = (int32_t)((pc + pm) / 2);
            }
            r.used_cpu = used_cpu;
            r.used_mem = used_mem;
            a.rows[t] = r;
        }
        if (f.used && lane < R) f.used[(uint64_t)t * R + lane] = s_used[lane];
    }
}

// One thread per pod: the four refusal words over the templates, staged SU_CHUNK at a time (F, labels, node_free); the
// rule word of (the pod's class, t) is read from global memory.  No atomics: each thread owns its pod's words.
template <int W>
__global__ void __launch_bounds__(SU_THREADS) k_fit_scaleup_reasons(PodView pv, ScaleupArgs a, FitScaleupArgs f) {
    __shared__ int64_t s_fc[SU_CHUNK], s_fm[SU_CHUNK];
    __shared__ uint64_t s_lab[W][SU_CHUNK];
    __shared__ int64_t s_nf[KS_BIND_MAX_RESOURCES][SU_CHUNK];
    const uint32_t p = blockIdx.x * SU_THREADS + threadIdx.x;
    const uint32_t R = f.R, T = a.T;
    const bool live = p < pv.P;
    const int64_t rc = live ? pv.req_cpu[p] : 0, rm = live ? pv.req_mem[p] : 0;
    uint64_t sel[W];
#pragma unroll
    for (int w = 0; w < W; w++) sel[w] = live ? pv.sel[(uint64_t)p * W + w] : 0;
    int64_t q[KS_BIND_MAX_RESOURCES];
    uint32_t rmask = 0;
#pragma unroll
    for (int r = 0; r < (int)KS_BIND_MAX_RESOURCES; r++) {
        q[r] = live && r < (int)R ? f.req[(uint64_t)p * R + r] : 0;
        rmask |= (q[r] != 0 ? 1u : 0u) << r;
    }
    const uint32_t* const rrow = f.nrules + (uint64_t)__ldg(f.ncls + (live ? f.group[p] : -1) + 1) * T;
    uint32_t word[5] = {0, 0, 0, 0, 0};
    for (uint32_t t0 = 0; t0 < T; t0 += SU_CHUNK) {
        const uint32_t n = min((uint32_t)SU_CHUNK, T - t0);
        __syncthreads();
        if (threadIdx.x < n) {
            const uint32_t t = t0 + threadIdx.x;
            s_fc[threadIdx.x] = a.free_cpu[t];
            s_fm[threadIdx.x] = a.free_mem[t];
#pragma unroll
            for (int w = 0; w < W; w++) s_lab[w][threadIdx.x] = a.labels[(uint64_t)t * W + w];
            for (uint32_t r = 0; r < R; r++) s_nf[r][threadIdx.x] = f.node_free[(uint64_t)r * T + t];
        }
        __syncthreads();
        if (!live) continue;
        for (uint32_t j = 0; j < n; j++) {
            uint64_t lab[W];
#pragma unroll
            for (int w = 0; w < W; w++) lab[w] = s_lab[w][j];
            const uint32_t s = fsu_stage<W>(rc, rm, sel, s_fc[j], s_fm[j], lab, q, rmask,
                                            [&](int r) { return s_nf[r][j]; }, __ldg(rrow + t0 + j));
            word[0] += s == 0;
            word[1] += s == 1;
            word[2] += s == 2;
            word[3] += s == 3;
        }
    }
    if (live) reinterpret_cast<uint4*>(f.refused)[p] = make_uint4(word[0], word[1], word[2], word[3]);
}

cudaError_t launch_fit_scaleup(const PodView& pv, uint32_t W, const ScaleupArgs& a, const FitScaleupArgs& f,
                               cudaStream_t st) {
    if (a.T == 0 || pv.P == 0) return cudaSuccess;
    const size_t smem = (size_t)(2 + f.R) * KS_SCALEUP_MAX_NODES * sizeof(int64_t); // 80 KiB at R = 8
    return with_label_width(W, [&](auto w) {
        constexpr int W_ = decltype(w)::value;
        cudaError_t e = cudaFuncSetAttribute(k_fit_scaleup_pack<W_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        k_fit_scaleup_pack<W_><<<a.slots, SU_THREADS, smem, st>>>(pv, a, f);
        g_launches++;
        e = cudaGetLastError();
        if (e != cudaSuccess || !f.refused) return e;
        k_fit_scaleup_reasons<W_><<<(pv.P + SU_THREADS - 1) / SU_THREADS, SU_THREADS, 0, st>>>(pv, a, f);
        g_launches++;
        return cudaGetLastError();
    });
}

uint32_t scaleup_slots(uint32_t T, int sms) { return std::min<uint32_t>(T, 4u * (uint32_t)std::max(sms, 1)); }

cudaError_t launch_scaleup(const PodView& pv, uint32_t W, const ScaleupArgs& a, cudaStream_t st) {
    if (a.T == 0 || pv.P == 0) return cudaSuccess;
    return with_label_width(W, [&](auto w) {
        constexpr int W_ = decltype(w)::value;
        k_scaleup_pack<W_><<<a.slots, SU_THREADS, 0, st>>>(pv, a);
        g_launches++;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess || !a.reasons) return e;
        k_scaleup_reasons<W_><<<(pv.P + SU_THREADS - 1) / SU_THREADS, SU_THREADS, 0, st>>>(pv, a);
        g_launches++;
        return cudaGetLastError();
    });
}

} // namespace ks
