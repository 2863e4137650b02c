// ks_internal.cuh — shared device-side views, PTX helpers and launch plumbing (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <type_traits>

#include "../../include/ksched.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libksched is written for sm_90a (H100)"
#endif

namespace ks {

constexpr int TILE_N = 1024;        // nodes per shared-memory tile of the direct kernel
constexpr int DIRECT_THREADS = 256; // 8 warps

// Device-resident node table (SoA, padded to a multiple of TILE_N with never-feasible sentinels:
// free = INT64_MIN, labels = 0).  labels are word-major: labels[w*Npad + n].
struct NodeTable {
    const int64_t* free_cpu;
    const int64_t* free_mem;
    const int64_t* alloc_cpu;
    const int64_t* alloc_mem;
    const uint64_t* labels;
    uint32_t N, Npad, W;
};

struct PodView {
    const int64_t* req_cpu;
    const int64_t* req_mem;
    const uint64_t* sel; // row-major [P*W]
    uint32_t P;
};

struct OutView {
    int32_t* node_idx;
    int64_t* score;
    uint32_t* cnt;
    uint32_t* mask;          // may be nullptr
    uint64_t mask_row_words; // row pitch in 32-bit words
    uint32_t mask_valid_words; // words per row that may be written: 8*ceil(N/256)
};

// Fused all-gather of the bindings (ks_exchange, include/ksched.h): peer-mapped destinations of this rank's shard
struct PeerOut {
    uint32_t n = 0; // peers; 0 = no exchange
    uint32_t world = 1, rank = 0;
    int32_t* idx[KS_MAX_PEERS];
    int64_t* score[KS_MAX_PEERS];
    uint32_t* flag[KS_MAX_PEERS];
    uint32_t* local_flags = nullptr;
    uint32_t* state = nullptr; // [0] = step sequence number, [1] = CTA completion counter, [2..11] = stamps (below)
};

// Diagnostic trace of the last exchange step: %globaltimer (ns) of 0 = first argmax CTA started, 1 = flags published,
// 2 = wait kernel started, 3 = wait kernel saw every peer, 4 = first CTA of the tail kernel started.  Five 64-bit words
// after the two state words.
__device__ __forceinline__ void exchange_stamp(const PeerOut& po, int which) {
    if (po.n == 0) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    reinterpret_cast<volatile unsigned long long*>(po.state + 2)[which] = t;
}

// Last CTA of the kernel that completes this rank's bindings: publish a new sequence number to every peer.
// Call at the very end of the kernel, by all threads of the CTA.
__device__ __forceinline__ void exchange_signal(const PeerOut& po) {
    if (po.n == 0) return;
    __syncthreads(); // every store of this CTA has been issued
    if (threadIdx.x == 0) {
        __threadfence_system(); // ... and is visible system-wide before the counter moves
        const uint32_t ctas = gridDim.x * gridDim.y * gridDim.z;
        if (atomicAdd(po.state + 1, 1u) == ctas - 1) {
            po.state[1] = 0; // every CTA has arrived: ready for the next launch
            const uint32_t seq = po.state[0] + 1;
            po.state[0] = seq;
            exchange_stamp(po, 1);
            __threadfence_system();
            for (uint32_t k = 0; k < po.n; k++)
                asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(po.flag[k]), "r"(seq) : "memory");
            asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(po.local_flags + po.rank), "r"(seq) : "memory");
        }
    }
}

// Per-(chunk,pod) partial results when the node dimension is split across CTAs (small P).
struct PartialView {
    int64_t* key;  // best policy key (LEFTOVER: node priority; LEAST_ALLOCATED, MOST_ALLOCATED: score)
    int32_t* idx;
    uint32_t* cnt;
};

extern std::atomic<uint64_t> g_launches;
// Every reallocation of a device buffer bumps this counter; it is part of the CUDA-graph cache key of ks_select, so a
// cached graph is never replayed after one of the buffers its nodes point to has moved (staging buffers grown by a
// larger call, ks_check_cells / ks_select_sampling scratch, the bit-parallel index, ...).
extern std::atomic<uint64_t> g_devbuf_epoch;

// ---- scores and the tie rule: one definition for every argmax path ----
// KS_SCORE_LEFTOVER: score = (free_cpu - rc) * 2^22 + (free_mem - rm) = node key - pod key.  The node key alone orders
// the nodes for a fixed pod; the range limits of ksched.h keep both keys and their difference inside int64.
__device__ __forceinline__ int64_t leftover_key(int64_t cpu, int64_t mem) {
    return (int64_t)(((uint64_t)cpu << 22) + (uint64_t)mem);
}
__device__ __forceinline__ int64_t leftover_score(int64_t node_key, int64_t rc, int64_t rm) {
    return node_key - leftover_key(rc, rm);
}
// KS_SCORE_LEAST_ALLOCATED in exact integer arithmetic: the mean of the truncated percentages left free after placement
__device__ __forceinline__ int64_t least_alloc_int(int64_t fc, int64_t fm, int64_t ac, int64_t am, int64_t rc, int64_t rm) {
    const int64_t pc = ac > 0 ? ((fc - rc) * 100) / ac : 0;
    const int64_t pm = am > 0 ? ((fm - rm) * 100) / am : 0;
    return (pc + pm) / 2;
}
// KS_SCORE_MOST_ALLOCATED in exact integer arithmetic: the mean of the truncated percentages requested after placement,
// requested = A - (f - q) clamped to [0, A].  Inside the limits of ksched.h every intermediate fits int64 (A - (f - q)
// is below 2^57 in magnitude and the clamped product below 100 * 2^55), and the score lies in [0, 100].
__device__ __forceinline__ int64_t most_alloc_term(int64_t f, int64_t a, int64_t q) {
    if (a <= 0) return 0;
    const int64_t u = a - (f - q);
    return (u < 0 ? 0 : u > a ? a : u) * 100 / a;
}
__device__ __forceinline__ int64_t most_alloc_int(int64_t fc, int64_t fm, int64_t ac, int64_t am, int64_t rc, int64_t rm) {
    return (most_alloc_term(fc, ac, rc) + most_alloc_term(fm, am, rm)) / 2;
}
// The balanced term of KS_SCORE_LEAST_BALANCED (upstream NodeResourcesBalancedAllocation, include/ksched.h): the shares
// x_r = u_r / A_r requested after placement, u_r clamped as in most_alloc_term, and trunc((1 - |x_c - x_m| / 2) * 100).
// Every step is one correctly rounded double operation spelled as an intrinsic, so no flag can contract it to an FMA or
// turn the division into a reciprocal: every kernel, and the restatement in the tests, gets the same bits.  In [0, 100].
__device__ __forceinline__ int64_t balanced_int(int64_t fc, int64_t fm, int64_t ac, int64_t am, int64_t rc, int64_t rm) {
    if (ac <= 0 || am <= 0) return 100; // a resource is skipped: std = 0
    int64_t uc = ac - (fc - rc), um = am - (fm - rm);
    uc = uc < 0 ? 0 : uc > ac ? ac : uc;
    um = um < 0 ? 0 : um > am ? am : um;
    const double xc = __ddiv_rn(__ll2double_rn(uc), __ll2double_rn(ac));
    const double xm = __ddiv_rn(__ll2double_rn(um), __ll2double_rn(am));
    const double sd = __ddiv_rn(fabs(__dsub_rn(xc, xm)), 2.0);
    return __double2ll_rz(__dmul_rn(__dsub_rn(1.0, sd), 100.0));
}
__device__ __forceinline__ int64_t least_balanced_int(int64_t fc, int64_t fm, int64_t ac, int64_t am, int64_t rc, int64_t rm) {
    return least_alloc_int(fc, fm, ac, am, rc, rm) + balanced_int(fc, fm, ac, am, rc, rm);
}
// The score of a policy that reads the allocatables, chosen at compile time: MOST_ALLOCATED, LEAST_BALANCED, else
// LEAST_ALLOCATED
template <int POLICY>
__device__ __forceinline__ int64_t alloc_score(int64_t fc, int64_t fm, int64_t ac, int64_t am, int64_t rc, int64_t rm) {
    return POLICY == KS_SCORE_MOST_ALLOCATED   ? most_alloc_int(fc, fm, ac, am, rc, rm)
           : POLICY == KS_SCORE_LEAST_BALANCED ? least_balanced_int(fc, fm, ac, am, rc, rm)
                                               : least_alloc_int(fc, fm, ac, am, rc, rm);
}
// The same chain with the policy chosen at run time, for the kernels that take it as an argument (k_stream_batch,
// k_gang_batch: one instantiation per label width).  LEFTOVER gives the node key; node n's allocatables are read only by
// the policies that score them.  The array pointers come by reference, so the kernel argument itself is read inside the
// branch that uses it, as in the chain written out in place: the kernels' code stays the same.
__device__ __forceinline__ int64_t alloc_score_rt(int policy, int64_t fc, int64_t fm, const int64_t* const& alloc_cpu,
                                                  const int64_t* const& alloc_mem, uint32_t n, int64_t rc, int64_t rm) {
    return policy == KS_SCORE_LEFTOVER ? leftover_key(fc, fm)
           : policy == KS_SCORE_MOST_ALLOCATED
               ? most_alloc_int(fc, fm, __ldg(alloc_cpu + n), __ldg(alloc_mem + n), rc, rm)
           : policy == KS_SCORE_LEAST_BALANCED
               ? least_balanced_int(fc, fm, __ldg(alloc_cpu + n), __ldg(alloc_mem + n), rc, rm)
               : least_alloc_int(fc, fm, __ldg(alloc_cpu + n), __ldg(alloc_mem + n), rc, rm);
}
// The score of a winning key: LEFTOVER's key is the node part only, every other policy's key is its score
template <int POLICY>
__device__ __forceinline__ int64_t key_score(int64_t key, int64_t rc, int64_t rm) {
    return POLICY == KS_SCORE_LEFTOVER ? leftover_score(key, rc, rm) : key;
}
// ... and with the policy chosen at run time, pod p's request read only for LEFTOVER
__device__ __forceinline__ int64_t key_score_rt(int policy, int64_t key, const int64_t* const& req_cpu,
                                                const int64_t* const& req_mem, uint32_t p) {
    return policy == KS_SCORE_LEFTOVER ? leftover_score(key, __ldg(req_cpu + p), __ldg(req_mem + p)) : key;
}
// Warp argmax over (key, idx) with idx < 0 for "no candidate": larger key wins, ties go to the lower node index.
// Every lane ends with the result.
__device__ __forceinline__ void warp_argmax(int64_t& key, int32_t& idx) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const int64_t ok = __shfl_xor_sync(0xffffffffu, key, off);
        const int32_t oi = __shfl_xor_sync(0xffffffffu, idx, off);
        const bool take = oi >= 0 && (idx < 0 || ok > key || (ok == key && oi < idx));
        if (take) {
            key = ok;
            idx = oi;
        }
    }
}
// Ordered merge of partial results over disjoint node ranges: fed in ascending range order, the strict '>' keeps the
// lower node index on ties.
__device__ __forceinline__ void merge_partial(int64_t& key, int32_t& idx, int64_t ok, int32_t oi) {
    if (oi >= 0 && (idx < 0 || ok > key)) {
        key = ok;
        idx = oi;
    }
}
// The same total order as a predicate: entry a ranks above entry b when a is an entry (ai >= 0) and b is empty, or a has
// the larger key, or the same key and the lower node index.
__device__ __forceinline__ bool topk_beats(int64_t ak, int32_t ai, int64_t bk, int32_t bi) {
    return ai >= 0 && (bi < 0 || ak > bk || (ak == bk && ai < bi));
}
// A ranked list held across the warp (ks_select_topk): lane j holds the j-th best (key, idx) for j < k, empty slots
// (idx = -1) come last and lanes >= k stay empty.  Inserts the warp-uniform candidate (ck, ci) at its rank, shifting the
// entries below it down one lane; a candidate that ranks k-th or lower changes nothing.  Called by the whole warp.
__device__ __forceinline__ void warp_topk_insert(int64_t& key, int32_t& idx, int64_t ck, int32_t ci, uint32_t k) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t pos = __popc(__ballot_sync(0xffffffffu, topk_beats(key, idx, ck, ci)));
    const int64_t uk = __shfl_up_sync(0xffffffffu, key, 1);
    const int32_t ui = __shfl_up_sync(0xffffffffu, idx, 1);
    if (lane < k && lane >= pos) {
        key = lane == pos ? ck : uk;
        idx = lane == pos ? ci : ui;
    }
}
// Priority preemption (ks_preempt): a candidate node as one 128-bit key (hi, lo) whose unsigned order is the plan's node
// order - the victims' highest priority, then their priority sum, then their count, then the node index, lowest first.
// hi = (max priority + 2^31) << 32 | sum >> 8 and lo = (sum & 255) << 56 | count << 48 | node, which is exact because
// the sum of at most 128 values below 2^32 stays below 2^39.  "No candidate" is (~0, ~0), above every key.
constexpr uint64_t PREEMPT_NONE = ~0ull;
__device__ __forceinline__ void preempt_key(int32_t vmax, int64_t vsum, uint32_t vcnt, uint32_t node, uint64_t& hi,
                                            uint64_t& lo) {
    hi = ((uint64_t)((uint32_t)vmax ^ 0x80000000u) << 32) | ((uint64_t)vsum >> 8);
    lo = ((uint64_t)vsum << 56) | ((uint64_t)vcnt << 48) | node;
}
__device__ __forceinline__ bool preempt_less(uint64_t ahi, uint64_t alo, uint64_t bhi, uint64_t blo) {
    return ahi < bhi || (ahi == bhi && alo < blo);
}
// Warp minimum of the keys above; every lane ends with the result.
__device__ __forceinline__ void warp_preempt_min(uint64_t& hi, uint64_t& lo) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const uint64_t oh = __shfl_xor_sync(0xffffffffu, hi, off);
        const uint64_t ol = __shfl_xor_sync(0xffffffffu, lo, off);
        if (preempt_less(oh, ol, hi, lo)) {
            hi = oh;
            lo = ol;
        }
    }
}

// Label-width dispatch: calls f(std::integral_constant<int, W>{}) for W in {1, 2, 4, 8}; any other W is invalid.
template <class F>
cudaError_t with_label_width(uint32_t W, F&& f) {
    switch (W) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 8: return f(std::integral_constant<int, 8>{});
        default: return cudaErrorInvalidValue;
    }
}

// The score policies (include/ksched.h).  A new policy is added here, in with_policy, in alloc_score / alloc_score_rt,
// in prepare_direct's list and in the tests' restatement (DESIGN.md 5j); every launcher reaches it through with_policy.
inline bool policy_valid(int policy) {
    return policy == KS_SCORE_LEFTOVER || policy == KS_SCORE_LEAST_ALLOCATED || policy == KS_SCORE_MOST_ALLOCATED ||
           policy == KS_SCORE_LEAST_BALANCED;
}
// Policy dispatch: calls f(std::integral_constant<int, POLICY>{}) for a valid policy; any other value is invalid.
template <class F>
cudaError_t with_policy(int policy, F&& f) {
    if (!policy_valid(policy)) return cudaErrorInvalidValue;
    switch (policy) {
        case KS_SCORE_LEFTOVER: return f(std::integral_constant<int, KS_SCORE_LEFTOVER>{});
        case KS_SCORE_LEAST_ALLOCATED: return f(std::integral_constant<int, KS_SCORE_LEAST_ALLOCATED>{});
        case KS_SCORE_MOST_ALLOCATED: return f(std::integral_constant<int, KS_SCORE_MOST_ALLOCATED>{});
        default: return f(std::integral_constant<int, KS_SCORE_LEAST_BALANCED>{});
    }
}

// ---- PTX helpers: mbarrier + 1-D TMA bulk copy (cp.async.bulk -> SASS UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes multiple of 16, 16B-aligned)
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// the same with an L2 cache policy (createpolicy) for the source lines
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}

// ---- launch-side plumbing shared by the API and the kernel files ----
// Arrays packed into one allocation in call order: take<T>(n) places n Ts at the next multiple of `align` and returns
// their byte offset; size is the bytes used so far.
struct BlockLayout {
    size_t size = 0;
    template <class T>
    size_t take(size_t n, size_t align = alignof(T)) {
        const size_t off = (size + align - 1) / align * align;
        size = off + n * sizeof(T);
        return off;
    }
};
template <class T>
T* at(void* base, size_t off) {
    return reinterpret_cast<T*>(static_cast<unsigned char*>(base) + off);
}

// Grow-only buffer in device (DevBuf) or pinned host (HostBuf) memory: ensure() reallocates, dropping the contents, when a
// call needs more than it holds.  Freed by its destructor, which must run with the owner's device current.
template <bool Pinned>
struct Buf {
    void* p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    void release() {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        release();
        if (!Pinned) g_devbuf_epoch++; // a pinned block leaves the epoch alone: no captured graph points into one
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = Pinned ? cudaHostAlloc(&p, want, cudaHostAllocDefault) : cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T>
    T* as() const {
        return static_cast<T*>(p);
    }
};
using DevBuf = Buf<false>;
using HostBuf = Buf<true>;

// Owner of one CUDA stream, event, graph or graph exec: Destroy runs when the owner goes (with its device current) or
// when reset() replaces the handle.  Created in place through &h; reads as the plain handle.
template <class H, cudaError_t (*Destroy)(H)>
struct Handle {
    H h = nullptr;
    Handle() = default;
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
    ~Handle() { reset(); }
    void reset() {
        if (h) Destroy(h);
        h = nullptr;
    }
    operator H() const { return h; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Graph = Handle<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Handle<cudaGraphExec_t, cudaGraphExecDestroy>;

struct SelectLaunch {
    NodeTable nt;
    PodView pv;
    OutView ov;
    int policy;
    cudaStream_t stream;
    // host-space outputs: when set, the launcher may copy these results back as soon as they exist (the bindings
    // are ready long before the mask kernel ends) and clears the pointer it has served
    int32_t* host_node_idx = nullptr;
    int64_t* host_score = nullptr;
    cudaEvent_t ready_event = nullptr; // caller's "bindings are final" event (ks_bindings.bindings_ready_event)
    PeerOut po;                        // fused all-gather of the bindings (po.n == 0: none)
};

} // namespace ks
