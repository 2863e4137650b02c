// ks_direct.cu — per-cell ("direct") kernels for sm_90a.
//   K0  k_node_free_reduce     free = alloc - sum(bound)            /root/reference/src/predicates.rs:27-38
//   K1  k_check_cells          2-bit reason code per cell           /root/reference/src/predicates.rs:63-77
//   K2d k_select_direct        fused feasible mask + count + argmax score, warp ballot packs 32 cells into
//                              one mask word, warp-shuffle argmax
//   K2e k_explain_counts       per-pod rejection counts (ks_explain)
//   K2k k_select_topk          per-pod ranked list of the k best feasible nodes (ks_select_topk), held across the warp
//   K2p k_preempt_scan         per-pod best preemption candidate (ks_preempt) over a per-call victim index;
//       k_preempt_emit         chunk merge, victim list and ks_preemption row
//   K2q k_fit_preempt_scan     the same under the full filter (ks_fit_preempt): rule words, scalar resources, pod count;
//       k_fit_preempt_emit     its merge, victim list, row and unresolvable count
//   K2u k_fit_drain_scan       ks_drain_check's scan under the full filter (ks_fit_drain_check), and its refusal pass;
//       k_fit_drain_commit     its commit, with the overlay's resource columns
// K2d, K2e, K2k, K2p and K2q share one node-tile scan (scan_node_tiles): tiles staged through shared memory by TMA bulk
// copies (cp.async.bulk + mbarrier), one lane per node, several pods per warp in registers.
// The per-cell kernel is the generic path (any score policy, any P); ks_bitpar.cu holds the bit-parallel
// fast path that the headline configuration uses.
#include "ks_internal.cuh"
#include "ks_launch.h"

#include <algorithm>

namespace ks {

std::atomic<uint64_t> g_launches{0};
std::atomic<uint64_t> g_devbuf_epoch{0};

// ------------------------------------------------------------------------------------------------ K0
__global__ void k_node_free_reduce(int64_t* __restrict__ free_cpu, int64_t* __restrict__ free_mem,
                                   const int32_t* __restrict__ bnode, const int64_t* __restrict__ bcpu,
                                   const int64_t* __restrict__ bmem, uint64_t B) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < B; i += stride) {
        int32_t n = bnode[i];
        // integer adds commute -> result is deterministic regardless of atomic order (util.rs:31-36)
        atomicAdd(reinterpret_cast<unsigned long long*>(free_cpu + n), (unsigned long long)(-bcpu[i]));
        atomicAdd(reinterpret_cast<unsigned long long*>(free_mem + n), (unsigned long long)(-bmem[i]));
    }
}

cudaError_t launch_free_reduce(int64_t* free_cpu, int64_t* free_mem, const int32_t* bnode, const int64_t* bcpu,
                               const int64_t* bmem, uint64_t B, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    int threads = 256;
    uint64_t blocks = (B + threads - 1) / threads;
    if (blocks > 4096) blocks = 4096; // grid-stride beyond that
    k_node_free_reduce<<<(unsigned)blocks, threads, 0, st>>>(free_cpu, free_mem, bnode, bcpu, bmem, B);
    g_launches++;
    return cudaGetLastError();
}

// range check of free values + static node priority for KS_SCORE_LEFTOVER: prio = free_cpu*2^22 + free_mem
__global__ void k_node_prio(const int64_t* __restrict__ free_cpu, const int64_t* __restrict__ free_mem,
                            int64_t* __restrict__ prio, uint32_t N, uint32_t Npad, int* __restrict__ range_flag) {
    uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= Npad) return;
    if (n >= N) {
        prio[n] = INT64_MIN;
        return;
    }
    int64_t fc = free_cpu[n], fm = free_mem[n];
    const int64_t LC = KS_MAX_CPU_MILLI, LM = KS_MAX_MEM_BYTES; // keeps prio and (free-req)*100 inside int64
    if (fc > LC || fc < -LC || fm > LM || fm < -LM) {
        atomicExch(range_flag, 1);
        prio[n] = INT64_MIN + 1;
        return;
    }
    prio[n] = leftover_key(fc, fm); // no overflow inside the range checked above: the same bits as fc * 2^22 + fm
}

cudaError_t launch_node_prio(const int64_t* free_cpu, const int64_t* free_mem, int64_t* prio, uint32_t N,
                             uint32_t Npad, int* range_flag, cudaStream_t st) {
    k_node_prio<<<(Npad + 255) / 256, 256, 0, st>>>(free_cpu, free_mem, prio, N, Npad, range_flag);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ exchange
// ks_exchange (include/ksched.h).  The bit-parallel path stores the bindings into the peers' gather buffers from
// inside its argmax kernels (ks_bitpar.cu); the per-cell path pushes its finished arrays with this kernel.
__global__ void __launch_bounds__(256)
    k_exchange_push(PeerOut po, const int32_t* __restrict__ node_idx, const int64_t* __restrict__ score, uint32_t P) {
    if (blockIdx.x == 0 && threadIdx.x == 0) exchange_stamp(po, 0);
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
        const int32_t ix = node_idx[p];
        const int64_t sc = score[p];
        for (uint32_t k = 0; k < po.n; k++) {
            po.idx[k][p] = ix;
            po.score[k][p] = sc;
        }
    }
    exchange_signal(po);
}

// One warp; lane r waits until rank r's flag carries this rank's current sequence number (all ranks step in
// lockstep).  A peer that never arrives raises *error_flag after ~4 s instead of hanging the GPU.
__global__ void __launch_bounds__(32) k_exchange_wait(PeerOut po, int* __restrict__ error_flag) {
    const uint32_t r = threadIdx.x;
    if (r == 0) exchange_stamp(po, 2);
    if (r < po.world && r != po.rank) {
        const uint32_t target = *reinterpret_cast<volatile uint32_t*>(po.state);
        unsigned long long t0;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        for (;;) {
            uint32_t v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(po.local_flags + r) : "memory");
            if ((int32_t)(v - target) >= 0) break;
            unsigned long long t1;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            if (t1 - t0 > 4000000000ull) {
                if (error_flag) atomicExch(error_flag, 2);
                break;
            }
            __nanosleep(200);
        }
    }
    __syncwarp();
    if (r == 0) exchange_stamp(po, 3);
}

cudaError_t launch_exchange_push(const PeerOut& po, const int32_t* node_idx, const int64_t* score, uint32_t P, cudaStream_t st) {
    if (po.n == 0) return cudaSuccess;
    const uint32_t grid = std::max(1u, std::min<uint32_t>(256u, (P + 255u) / 256u));
    k_exchange_push<<<grid, 256, 0, st>>>(po, node_idx, score, P);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_exchange_wait(const PeerOut& po, int* error_flag, cudaStream_t st) {
    if (po.n == 0) return cudaSuccess;
    k_exchange_wait<<<1, 32, 0, st>>>(po, error_flag);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ store ceiling
// What a kernel that ONLY writes can reach on this device (ks_measure_write_bandwidth): 128-bit stores (the widest sm_90
// has), consecutive lanes on consecutive 16 bytes, grid-stride, nothing else.  The mask kernel is compared with this next
// to the copy-based HBM peak (DESIGN.md section 7).
__global__ void __launch_bounds__(256) k_fill256(uint8_t* __restrict__ dst, uint64_t n32, uint32_t v) {
    const uint64_t n16 = 2 * n32;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (uint64_t)gridDim.x * blockDim.x)
        asm volatile("st.global.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst + i * 16), "r"(v) : "memory");
}

cudaError_t launch_fill256(void* dst, uint64_t bytes, uint32_t v, int sms, cudaStream_t st) {
    k_fill256<<<sms * 8, 256, 0, st>>>(static_cast<uint8_t*>(dst), bytes / 32, v);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ K1
__device__ __forceinline__ int cell_code(int64_t rc, int64_t rm, const uint64_t* __restrict__ sel, int64_t fc,
                                         int64_t fm, const uint64_t* __restrict__ labels, uint32_t n,
                                         uint32_t Npad, uint32_t W) {
    bool fit = (rc <= fc) && (rm <= fm); // predicates.rs:42
    uint64_t miss = 0;
    for (uint32_t w = 0; w < W; w++) miss |= sel[w] & ~labels[(uint64_t)w * Npad + n];
    return !fit ? KS_CELL_NOT_ENOUGH_RESOURCES : (miss ? KS_CELL_NODE_SELECTOR_MISMATCH : KS_CELL_OK); // :68-76
}

__global__ void k_check_cells(NodeTable nt, PodView pv, uint8_t* __restrict__ codes, uint32_t node_begin,
                              uint32_t node_count) {
    uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t total = (uint64_t)pv.P * node_count;
    if (cell >= total) return;
    uint32_t p = (uint32_t)(cell / node_count);
    uint32_t n = node_begin + (uint32_t)(cell % node_count);
    codes[cell] = (uint8_t)cell_code(pv.req_cpu[p], pv.req_mem[p], pv.sel + (uint64_t)p * nt.W, nt.free_cpu[n],
                                     nt.free_mem[n], nt.labels, n, nt.Npad, nt.W);
}

cudaError_t launch_check_cells(const NodeTable& nt, const PodView& pv, uint8_t* codes, uint32_t node_begin,
                               uint32_t node_count, cudaStream_t st) {
    uint64_t total = (uint64_t)pv.P * node_count;
    if (total == 0) return cudaSuccess;
    uint64_t blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    k_check_cells<<<(unsigned)blocks, 256, 0, st>>>(nt, pv, codes, node_begin, node_count);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ K1s
// The reference's own selection policy (/root/reference/src/main.rs:49-71) with a seeded generator: up to
// `attempts` uniform draws with replacement per pod, the first draw whose cell passes check_node_validity wins.
// One thread per pod; the node rows it touches are random gathers served by L2 (the node table is a few MB).
__device__ __forceinline__ uint64_t splitmix64_next(uint64_t& s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void k_select_sampling(NodeTable nt, PodView pv, uint32_t attempts, uint64_t seed, uint64_t pod_offset,
                                  int32_t* __restrict__ node_idx, uint32_t* __restrict__ n_attempts,
                                  int32_t* __restrict__ draw_node, uint8_t* __restrict__ draw_code) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pv.P) return;
    uint64_t state = KS_SAMPLING_STREAM(seed, pod_offset + p);
    const int64_t rc = pv.req_cpu[p], rm = pv.req_mem[p];
    const uint64_t* sel = pv.sel + (uint64_t)p * nt.W;
    int32_t chosen = -1;
    uint32_t a = 0;
    for (; a < attempts; a++) {                                         // main.rs:53
        const uint32_t n = (uint32_t)(splitmix64_next(state) % nt.N); // :56-57 choose()
        const int code = cell_code(rc, rm, sel, nt.free_cpu[n], nt.free_mem[n], nt.labels, n, nt.Npad, nt.W); // :61
        if (draw_node) draw_node[(uint64_t)p * attempts + a] = (int32_t)n;
        if (draw_code) draw_code[(uint64_t)p * attempts + a] = (uint8_t)code; // the reason main.rs:62 logs
        if (code == KS_CELL_OK) {                                     // :63-65
            chosen = (int32_t)n;
            a++;
            break;
        }
    }
    for (uint32_t r = a; r < attempts; r++) { // attempts never made
        if (draw_node) draw_node[(uint64_t)p * attempts + r] = -1;
        if (draw_code) draw_code[(uint64_t)p * attempts + r] = 0xff;
    }
    node_idx[p] = chosen;
    if (n_attempts) n_attempts[p] = a;
}

cudaError_t launch_select_sampling(const NodeTable& nt, const PodView& pv, uint32_t attempts, uint64_t seed,
                                   uint64_t pod_offset, int32_t* node_idx, uint32_t* n_attempts, int32_t* draw_node,
                                   uint8_t* draw_code, cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    k_select_sampling<<<(pv.P + 255) / 256, 256, 0, st>>>(nt, pv, attempts, seed, pod_offset, node_idx, n_attempts,
                                                          draw_node, draw_code);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ K2d / K2e
__host__ __device__ constexpr uint32_t pods_per_warp(uint32_t W) { return W <= 2 ? 8u : (W == 4 ? 4u : 2u); }

// Shared memory of one stage of the node-tile scan: free_cpu, free_mem, the W label words and, when the body scores
// LeastAllocated, alloc_cpu and alloc_mem, TILE_N nodes each.  Two stages double-buffer the tiles.
template <int W, bool ALLOC>
__host__ __device__ constexpr uint32_t tile_stage_bytes() {
    return (2u + W + (ALLOC ? 2u : 0u)) * TILE_N * 8u;
}
template <int W, bool ALLOC>
__host__ __device__ constexpr uint32_t tile_smem_bytes() {
    return 2u * tile_stage_bytes<W, ALLOC>();
}

// The first of this warp's PW pods.
template <int PW>
__device__ __forceinline__ uint32_t warp_first_pod() {
    return (blockIdx.x * (DIRECT_THREADS / 32) + (threadIdx.x >> 5)) * PW;
}

// This warp's pods p0.. into warp-uniform registers.  Slots past P repeat the last pod (their results are never
// written).
template <int W, int PW>
__device__ __forceinline__ void load_warp_pods(const PodView& pv, uint32_t p0, int64_t (&rc)[PW], int64_t (&rm)[PW],
                                               uint64_t (&sel)[PW][W]) {
#pragma unroll
    for (int i = 0; i < PW; i++) {
        const uint32_t p = min(p0 + i, pv.P - 1);
        rc[i] = __ldg(pv.req_cpu + p);
        rm[i] = __ldg(pv.req_mem + p);
#pragma unroll
        for (int w = 0; w < W; w++) sel[i][w] = __ldg(pv.sel + (uint64_t)p * W + w);
    }
}

// The node scan of K2d and K2e over this CTA's chunk of tiles, [blockIdx.y * tiles_per_chunk, +tiles_per_chunk).  One
// thread stages each tile through shared memory with bulk copies, one tile ahead of the warps.  The warp's first pod p0
// and its pods' registers rc/rm/sel are loaded while the first tile is in flight.  Each lane takes one node of every
// group of 32 and the whole warp calls cell(g, node, real, fc, fm, lab, ac, am), so the body may ballot; real is false
// for padding nodes, and ac/am are 0 unless ALLOC.  After a tile's 32 groups every thread calls tile_done(tile).
template <int W, bool ALLOC, int PW, class Cell, class TileDone>
__device__ __forceinline__ void scan_node_tiles(const NodeTable& nt, uint32_t tiles_per_chunk, const PodView& pv, uint32_t& p0,
                                                int64_t (&rc)[PW], int64_t (&rm)[PW], uint64_t (&sel)[PW][W], Cell&& cell,
                                                TileDone&& tile_done) {
    constexpr uint32_t STAGE_BYTES = tile_stage_bytes<W, ALLOC>();
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[2];

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t tile_begin = blockIdx.y * tiles_per_chunk;
    const uint32_t tile_end = min(tile_begin + tiles_per_chunk, nt.Npad / TILE_N);

    if (threadIdx.x == 0) {
        mbar_init(&full_bar[0], 1);
        mbar_init(&full_bar[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    auto issue_tile = [&](uint32_t tile, uint32_t stage) {
        // arm the barrier with the byte count, then issue one bulk copy per SoA column
        unsigned char* dst = smem_raw + (size_t)stage * STAGE_BYTES;
        uint64_t* bar = &full_bar[stage];
        mbar_arrive_expect_tx(bar, STAGE_BYTES);
        const size_t off = (size_t)tile * TILE_N;
        tma_bulk_g2s(dst, nt.free_cpu + off, TILE_N * 8, bar);
        tma_bulk_g2s(dst + TILE_N * 8, nt.free_mem + off, TILE_N * 8, bar);
#pragma unroll
        for (int w = 0; w < W; w++)
            tma_bulk_g2s(dst + (2 + w) * TILE_N * 8, nt.labels + (size_t)w * nt.Npad + off, TILE_N * 8, bar);
        if (ALLOC) {
            tma_bulk_g2s(dst + (2 + W) * TILE_N * 8, nt.alloc_cpu + off, TILE_N * 8, bar);
            tma_bulk_g2s(dst + (3 + W) * TILE_N * 8, nt.alloc_mem + off, TILE_N * 8, bar);
        }
    };

    if (threadIdx.x == 0 && tile_begin < tile_end) issue_tile(tile_begin, 0);
    p0 = warp_first_pod<PW>();
    load_warp_pods(pv, p0, rc, rm, sel);

    for (uint32_t tile = tile_begin; tile < tile_end; tile++) {
        const uint32_t it = tile - tile_begin, stage = it & 1;
        if (threadIdx.x == 0 && tile + 1 < tile_end) issue_tile(tile + 1, stage ^ 1);
        mbar_wait(&full_bar[stage], (it >> 1) & 1);

        const unsigned char* base = smem_raw + (size_t)stage * STAGE_BYTES;
        const int64_t* s_fc = reinterpret_cast<const int64_t*>(base);
        const int64_t* s_fm = s_fc + TILE_N;
        const uint64_t* s_lab = reinterpret_cast<const uint64_t*>(s_fm + TILE_N);
        const int64_t* s_ac = reinterpret_cast<const int64_t*>(s_lab + (size_t)W * TILE_N);
        const int64_t* s_am = s_ac + TILE_N;

#pragma unroll 2
        for (uint32_t g = 0; g < 32; g++) {
            const uint32_t ln = g * 32 + lane;
            const int64_t fc = s_fc[ln], fm = s_fm[ln];
            uint64_t lab[W];
#pragma unroll
            for (int w = 0; w < W; w++) lab[w] = s_lab[w * TILE_N + ln];
            const uint32_t node = tile * TILE_N + ln;
            cell(g, node, node < nt.N, fc, fm, lab, ALLOC ? s_ac[ln] : 0, ALLOC ? s_am[ln] : 0);
        }
        tile_done(tile);
        __syncthreads(); // everyone is done with `stage` before it is refilled two iterations later
    }
}

template <int W, int POLICY, bool EMIT_MASK>
__global__ void __launch_bounds__(DIRECT_THREADS)
    k_select_direct(NodeTable nt, PodView pv, OutView ov, PartialView part, uint32_t tiles_per_chunk) {
    constexpr int PW = pods_per_warp(W);
    constexpr bool ALLOC = POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    const uint32_t lane = threadIdx.x & 31;
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int64_t best[PW];
    int32_t bidx[PW];
    uint32_t cnt[PW];
    uint32_t acc[PW];
#pragma unroll
    for (int i = 0; i < PW; i++) {
        best[i] = INT64_MIN;
        bidx[i] = -1;
        cnt[i] = 0;
        acc[i] = 0;
    }

    scan_node_tiles<W, ALLOC>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t g, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t ac, int64_t am) {
            const int64_t key_n = ALLOC ? 0 : leftover_key(fc, fm); // LEFTOVER: node priority; the pod part is constant
#pragma unroll
            for (int i = 0; i < PW; i++) {
                const bool fit = (rc[i] <= fc) & (rm[i] <= fm);
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const bool ok = fit && (miss == 0) && real;
                const uint32_t b = __ballot_sync(0xffffffffu, ok);
                cnt[i] += __popc(b);
                if (EMIT_MASK) acc[i] = (lane == g) ? b : acc[i];
                if (ok) {
                    const int64_t key = ALLOC ? alloc_score<POLICY>(fc, fm, ac, am, rc[i], rm[i]) : key_n;
                    if (key > best[i]) {
                        best[i] = key;
                        bidx[i] = (int32_t)node;
                    }
                }
            }
        },
        [&](uint32_t tile) {
            if (!EMIT_MASK) return;
            const uint32_t word = tile * 32 + lane; // 32 words per 1024-node tile
            if (word < ov.mask_valid_words) {
#pragma unroll
                for (int i = 0; i < PW; i++)
                    if (p0 + i < pv.P) ov.mask[(uint64_t)(p0 + i) * ov.mask_row_words + word] = acc[i];
            }
        });

#pragma unroll
    for (int i = 0; i < PW; i++) {
        int64_t k = best[i];
        int32_t ix = bidx[i];
        warp_argmax(k, ix);
        if (lane == 0 && p0 + i < pv.P) {
            const uint32_t p = p0 + i;
            if (gridDim.y == 1) {
                const int64_t s = ix < 0 ? 0 : key_score<POLICY>(k, rc[i], rm[i]);
                if (ov.node_idx) ov.node_idx[p] = ix;
                if (ov.score) ov.score[p] = s;
                if (ov.cnt) ov.cnt[p] = cnt[i];
            } else {
                const uint64_t o = (uint64_t)blockIdx.y * pv.P + p;
                part.key[o] = k;
                part.idx[o] = ix;
                part.cnt[o] = cnt[i];
            }
        }
    }
}

// combine the partials of the node chunks, in ascending chunk order
template <int POLICY>
__global__ void k_select_combine(PodView pv, OutView ov, PartialView part, uint32_t n_chunks) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pv.P) return;
    int64_t k = INT64_MIN;
    int32_t ix = -1;
    uint32_t c = 0;
    for (uint32_t ch = 0; ch < n_chunks; ch++) {
        const uint64_t o = (uint64_t)ch * pv.P + p;
        c += part.cnt[o];
        merge_partial(k, ix, part.key[o], part.idx[o]);
    }
    const int64_t s = ix < 0 ? 0 : key_score<POLICY>(k, pv.req_cpu[p], pv.req_mem[p]);
    if (ov.node_idx) ov.node_idx[p] = ix;
    if (ov.score) ov.score[p] = s;
    if (ov.cnt) ov.cnt[p] = c;
}

// Per-pod rejection counts (ks_explain): three ballots per 32 nodes.  Counts of one CTA row are warp-uniform; with
// gridDim.y > 1 the node chunks add into a zeroed output, and integer adds make the result independent of their order.
template <int W>
__global__ void __launch_bounds__(DIRECT_THREADS)
    k_explain_counts(NodeTable nt, PodView pv, uint32_t* __restrict__ out, uint32_t tiles_per_chunk) {
    constexpr int PW = pods_per_warp(W);
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    uint32_t n_cpu[PW], n_mem[PW], n_res[PW], n_sel[PW];
#pragma unroll
    for (int i = 0; i < PW; i++) n_cpu[i] = n_mem[i] = n_res[i] = n_sel[i] = 0;

    scan_node_tiles<W, false>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t, uint32_t, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t, int64_t) {
#pragma unroll
            for (int i = 0; i < PW; i++) {
                const bool cpu_fail = real && rc[i] > fc; // predicates.rs:42, each half
                const bool mem_fail = real && rm[i] > fm;
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const bool sel_fail = real && !cpu_fail && !mem_fail && miss != 0; // fit first, :68-74
                const uint32_t bc = __ballot_sync(0xffffffffu, cpu_fail);
                const uint32_t bm = __ballot_sync(0xffffffffu, mem_fail);
                const uint32_t bs = __ballot_sync(0xffffffffu, sel_fail);
                n_cpu[i] += __popc(bc);
                n_mem[i] += __popc(bm);
                n_res[i] += __popc(bc | bm);
                n_sel[i] += __popc(bs);
            }
        },
        [](uint32_t) {});

    if ((threadIdx.x & 31) == 0) { // the counts are warp-uniform
#pragma unroll
        for (int i = 0; i < PW; i++) {
            if (p0 + i >= pv.P) continue;
            uint32_t* o = out + (uint64_t)(p0 + i) * 4;
            if (gridDim.y == 1) {
                o[0] = n_cpu[i];
                o[1] = n_mem[i];
                o[2] = n_res[i];
                o[3] = n_sel[i];
            } else {
                atomicAdd(o + 0, n_cpu[i]);
                atomicAdd(o + 1, n_mem[i]);
                atomicAdd(o + 2, n_res[i]);
                atomicAdd(o + 3, n_sel[i]);
            }
        }
    }
}

// Ranked candidates (ks_select_topk): per pod the k best feasible nodes, held across the warp (warp_topk_insert), plus
// the feasible count.  A feasible cell that ranks above the list's k-th entry (the threshold, warp-uniform) is a
// candidate.  Each group of 32 nodes takes one ballot of candidates and inserts them in ascending lane order, which is
// ascending node order; after each insertion the threshold is re-read and the candidates it now excludes are dropped.
// With gridDim.y > 1 each node chunk writes its list and count to partials [chunk][P][k], merged by k_topk_combine.
template <int W, int POLICY>
// One CTA per SM: eight lists per warp at W <= 2 need more than 128 registers, and ptxas spills when held to that.
__global__ void __launch_bounds__(DIRECT_THREADS, 1)
    k_select_topk(NodeTable nt, PodView pv, OutView ov, PartialView part, uint32_t k, uint32_t tiles_per_chunk) {
    constexpr int PW = pods_per_warp(W);
    constexpr bool ALLOC = POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    const uint32_t lane = threadIdx.x & 31;
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int64_t lkey[PW], tkey[PW]; // this lane's list entry; the k-th entry of the list
    int32_t lidx[PW], tidx[PW];
    uint32_t cnt[PW];
#pragma unroll
    for (int i = 0; i < PW; i++) {
        lkey[i] = tkey[i] = 0;
        lidx[i] = tidx[i] = -1;
        cnt[i] = 0;
    }

    scan_node_tiles<W, ALLOC>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t ac, int64_t am) {
            const int64_t key_n = ALLOC ? 0 : leftover_key(fc, fm); // LEFTOVER: node priority; the pod part is constant
#pragma unroll
            for (int i = 0; i < PW; i++) {
                const bool fit = (rc[i] <= fc) & (rm[i] <= fm);
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const bool ok = fit && (miss == 0) && real;
                cnt[i] += __popc(__ballot_sync(0xffffffffu, ok));
                const int64_t key = ALLOC ? (ok ? alloc_score<POLICY>(fc, fm, ac, am, rc[i], rm[i]) : 0) : key_n;
                uint32_t cand = __ballot_sync(0xffffffffu, ok && topk_beats(key, (int32_t)node, tkey[i], tidx[i]));
                while (cand) { // warp-uniform
                    const int src = __ffs(cand) - 1;
                    cand &= cand - 1;
                    const int64_t ck = __shfl_sync(0xffffffffu, key, src);
                    const int32_t ci = (int32_t)(node - lane + src);
                    warp_topk_insert(lkey[i], lidx[i], ck, ci, k);
                    tkey[i] = __shfl_sync(0xffffffffu, lkey[i], k - 1);
                    tidx[i] = __shfl_sync(0xffffffffu, lidx[i], k - 1);
                    cand &= __ballot_sync(0xffffffffu, topk_beats(key, (int32_t)node, tkey[i], tidx[i]));
                }
            }
        },
        [](uint32_t) {});

#pragma unroll
    for (int i = 0; i < PW; i++) {
        const uint32_t p = p0 + i;
        if (p >= pv.P) continue; // warp-uniform
        if (gridDim.y == 1) {
            const uint64_t o = (uint64_t)p * k + lane;
            if (lane < k) {
                ov.node_idx[o] = lidx[i];
                if (ov.score) ov.score[o] = lidx[i] < 0 ? 0 : key_score<POLICY>(lkey[i], rc[i], rm[i]);
            }
            if (lane == 0 && ov.cnt) ov.cnt[p] = cnt[i];
        } else {
            const uint64_t row = (uint64_t)blockIdx.y * pv.P + p;
            if (lane < k) {
                part.key[row * k + lane] = lkey[i];
                part.idx[row * k + lane] = lidx[i];
            }
            if (lane == 0) part.cnt[row] = cnt[i];
        }
    }
}

// Merge the chunk lists of k_select_topk, one warp per pod, in ascending chunk order; keys become scores.
template <int POLICY>
__global__ void __launch_bounds__(256) k_topk_combine(PodView pv, OutView ov, PartialView part, uint32_t n_chunks, uint32_t k) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (p >= pv.P) return; // warp-uniform
    int64_t key = 0, tkey = 0;
    int32_t idx = -1, tidx = -1;
    uint32_t c = 0;
    for (uint32_t ch = 0; ch < n_chunks; ch++) {
        const uint64_t row = (uint64_t)ch * pv.P + p;
        c += part.cnt[row];
        const int64_t pk = lane < k ? part.key[row * k + lane] : 0;
        const int32_t pi = lane < k ? part.idx[row * k + lane] : -1;
        for (uint32_t j = 0; j < k; j++) {
            const int64_t ck = __shfl_sync(0xffffffffu, pk, j);
            const int32_t ci = __shfl_sync(0xffffffffu, pi, j);
            if (!topk_beats(ck, ci, tkey, tidx)) break; // the chunk's list is ranked: nothing after j gets in either
            warp_topk_insert(key, idx, ck, ci, k);
            tkey = __shfl_sync(0xffffffffu, key, k - 1);
            tidx = __shfl_sync(0xffffffffu, idx, k - 1);
        }
    }
    const uint64_t o = (uint64_t)p * k + lane;
    if (lane < k) {
        ov.node_idx[o] = idx;
        if (ov.score)
            ov.score[o] = idx < 0 ? 0 : key_score<POLICY>(key, pv.req_cpu[p], pv.req_mem[p]);
    }
    if (lane == 0 && ov.cnt) ov.cnt[p] = c;
}

// ------------------------------------------------------------------------------------------------ K2p (ks_preempt)
// Steps 2-5 of ks_preempt (include/ksched.h) for one pod (priority pi, request rc/rm) on one node (free fc/fm, sorted
// segment [s0, s1) of the victim index): the lower set is the segment's prefix below pi (binary search), the room check
// reads its prefix sums, and the reprieve walk goes backwards from the prefix's end - priority descending, ties to the
// lower bound index.  Returns whether the node is a candidate, with the victims' highest priority, priority sum (each
// pi_b + 2^31) and count; when out is not null the victims' bound indices go to out[0..count).  The range rule of
// ks_preempt keeps every sum below inside int64.
__device__ __forceinline__ bool preempt_walk(const VictimIndex& vx, uint32_t s0, uint32_t s1, int32_t pi, int64_t rc,
                                             int64_t rm, int64_t fc, int64_t fm, uint32_t max_victims, int32_t& vmax,
                                             int64_t& vsum, uint32_t& vcnt, int32_t* out) {
    uint32_t lo = s0, hi = s1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(vx.prio + mid) < pi) lo = mid + 1;
        else hi = mid;
    }
    if (lo == s0) return false; // no pod of lower priority
    int64_t ac = fc + __ldg(vx.pre_cpu + lo - 1), am = fm + __ldg(vx.pre_mem + lo - 1);
    if (rc > ac || rm > am) return false; // evicting the whole lower set is not enough
    vmax = INT32_MIN;
    vsum = 0;
    vcnt = 0;
    for (uint32_t j = lo; j-- > s0;) {
        const int64_t bc = __ldg(vx.cpu + j), bm = __ldg(vx.mem + j);
        if (rc <= ac - bc && rm <= am - bm) { // still fits without evicting b: reprieved
            ac -= bc;
            am -= bm;
            continue;
        }
        if (vcnt == max_victims) return false;
        const int32_t bp = __ldg(vx.prio + j);
        if (vcnt == 0) vmax = bp; // visited in descending priority: the first victim has the highest
        if (out) out[vcnt] = (int32_t)__ldg(vx.idx + j);
        vsum += (int64_t)bp + 2147483648ll;
        vcnt++;
    }
    return true; // at least one victim: with none, the pod would fit free[] and the node would not be eligible
}

// Candidate scan (ks_preempt): per pod the feasible count (as K2d counts it), the number of candidate nodes and the
// best candidate's key (preempt_key).  A cell goes to preempt_walk only when it fails on resources, its selector matches
// and the node holds a pod of lower priority (min_prio, one coalesced load per node); the walk reads the node's segment
// from L2.  Results go to partials [blockIdx.y][P], merged by k_preempt_emit.
template <int W>
__global__ void __launch_bounds__(DIRECT_THREADS)
    k_preempt_scan(NodeTable nt, PodView pv, const int32_t* __restrict__ pod_prio, VictimIndex vx, uint32_t max_victims,
                   PreemptPartials part, uint32_t tiles_per_chunk) {
    constexpr int PW = pods_per_warp(W);
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int32_t pi[PW];
    uint64_t bhi[PW], blo[PW];
    uint32_t cnt[PW], ncand[PW];
    const uint32_t q0 = warp_first_pod<PW>(); // the p0 scan_node_tiles sets
#pragma unroll
    for (int i = 0; i < PW; i++) {
        pi[i] = __ldg(pod_prio + min(q0 + i, pv.P - 1));
        bhi[i] = blo[i] = PREEMPT_NONE;
        cnt[i] = ncand[i] = 0;
    }

    scan_node_tiles<W, false>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t, int64_t) {
            const int32_t mp = real ? __ldg(vx.min_prio + node) : INT32_MAX; // padding: never a candidate
#pragma unroll
            for (int i = 0; i < PW; i++) {
                const bool fit = (rc[i] <= fc) & (rm[i] <= fm);
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                cnt[i] += __popc(__ballot_sync(0xffffffffu, fit && (miss == 0) && real));
                if (!fit && miss == 0 && mp < pi[i]) {
                    int32_t vmax;
                    int64_t vsum;
                    uint32_t vcnt;
                    if (preempt_walk(vx, __ldg(vx.off + node), __ldg(vx.off + node + 1), pi[i], rc[i], rm[i], fc, fm,
                                     max_victims, vmax, vsum, vcnt, nullptr)) {
                        uint64_t h, l;
                        preempt_key(vmax, vsum, vcnt, node, h, l);
                        ncand[i]++;
                        if (preempt_less(h, l, bhi[i], blo[i])) {
                            bhi[i] = h;
                            blo[i] = l;
                        }
                    }
                }
            }
        },
        [](uint32_t) {});

#pragma unroll
    for (int i = 0; i < PW; i++) {
        uint64_t h = bhi[i], l = blo[i];
        warp_preempt_min(h, l);
        const uint32_t c = __reduce_add_sync(0xffffffffu, ncand[i]);
        const uint32_t p = p0 + i;
        if ((threadIdx.x & 31) == 0 && p < pv.P) {
            const uint64_t o = (uint64_t)blockIdx.y * pv.P + p;
            part.hi[o] = h;
            part.lo[o] = l;
            part.cand[o] = c;
            part.cnt[o] = cnt[i];
        }
    }
}

// One thread per pod: merge the node chunks in ascending order, apply "already fits => no plan", walk the chosen node
// once more to list the victims, and write the ks_preemption row.  n_chunks = 0 (no node) gives every pod no plan.
__global__ void __launch_bounds__(256)
    k_preempt_emit(NodeTable nt, PodView pv, const int32_t* __restrict__ pod_prio, VictimIndex vx, uint32_t max_victims,
                   PreemptPartials part, uint32_t n_chunks, ks_preemption* __restrict__ out, int32_t* __restrict__ victims) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pv.P) return;
    uint64_t hi = PREEMPT_NONE, lo = PREEMPT_NONE;
    uint32_t cand = 0, cnt = 0;
    for (uint32_t ch = 0; ch < n_chunks; ch++) {
        const uint64_t o = (uint64_t)ch * pv.P + p;
        cnt += part.cnt[o];
        cand += part.cand[o];
        if (preempt_less(part.hi[o], part.lo[o], hi, lo)) {
            hi = part.hi[o];
            lo = part.lo[o];
        }
    }
    ks_preemption r;
    r.node_idx = -1;
    r.n_victims = 0;
    r.candidates = cnt ? 0u : cand;
    r.feasible_cnt = cnt;
    r.max_victim_priority = INT32_MIN;
    r.reserved = 0;
    r.victim_priority_sum = 0;
    int32_t* v = victims ? victims + (uint64_t)p * max_victims : nullptr;
    if (cnt == 0 && hi != PREEMPT_NONE) {
        const uint32_t node = (uint32_t)(lo & 0xffffffffffffull);
        int32_t vmax;
        int64_t vsum;
        uint32_t vcnt;
        if (preempt_walk(vx, vx.off[node], vx.off[node + 1], pod_prio[p], pv.req_cpu[p], pv.req_mem[p],
                         nt.free_cpu[node], nt.free_mem[node], max_victims, vmax, vsum, vcnt, v)) {
            r.node_idx = (int32_t)node;
            r.n_victims = vcnt;
            r.max_victim_priority = vmax;
            r.victim_priority_sum = vsum;
        }
    }
    if (v)
        for (uint32_t j = r.n_victims; j < max_victims; j++) v[j] = -1;
    out[p] = r;
}

// ------------------------------------------------------------------------------------------------ K2q (ks_fit_preempt)
// preempt_walk with the R request columns (include/ksched.h, ks_fit_preempt steps 3-4): besides cpu and memory, every
// resource in rmask (the pod's non-zero requests req[r]; a zero request always fits) keeps its own avail, free_r[n] plus
// the lower set's prefix sum, and a bound pod is reprieved only when the pod still fits in every one of them.  The
// requested resources are listed once, 4 bits each in rlist, so each step of the walk costs one test per requested
// resource and one more; a pod that requests none walks as preempt_walk does.  The range rule of ks_fit_preempt keeps
// every sum inside int64.
__device__ __forceinline__ bool fit_preempt_walk(const VictimIndex& vx, const FitPreemptArgs& fa, uint32_t N,
                                                 uint32_t node, int32_t pi, int64_t rc, int64_t rm, int64_t fc,
                                                 int64_t fm, const int64_t* req, uint32_t rmask, uint32_t max_victims,
                                                 int32_t& vmax, int64_t& vsum, uint32_t& vcnt, int32_t* out) {
    const uint32_t s0 = __ldg(vx.off + node), s1 = __ldg(vx.off + node + 1);
    uint32_t lo = s0, hi = s1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(vx.prio + mid) < pi) lo = mid + 1;
        else hi = mid;
    }
    if (lo == s0) return false; // no pod of lower priority
    int64_t ac = fc + __ldg(vx.pre_cpu + lo - 1), am = fm + __ldg(vx.pre_mem + lo - 1);
    bool room = rc <= ac && rm <= am;
    const uint32_t nreq = __popc(rmask);
    uint32_t rlist = 0;
    for (uint32_t m = rmask, k = 0; m; m &= m - 1, k++) rlist |= (uint32_t)(__ffs(m) - 1) << (4 * k);
    int64_t ar[KS_BIND_MAX_RESOURCES];
#pragma unroll
    for (uint32_t k = 0; k < KS_BIND_MAX_RESOURCES; k++) {
        if (k == nreq) break;
        const uint32_t r = rlist >> (4 * k) & 15u;
        ar[k] = __ldg(fa.node_free + (size_t)r * N + node) + __ldg(fa.vpre + (size_t)r * fa.B + lo - 1);
        room &= req[r] <= ar[k];
    }
    if (!room) return false; // evicting the whole lower set is not enough
    vmax = INT32_MIN;
    vsum = 0;
    vcnt = 0;
    for (uint32_t j = lo; j-- > s0;) {
        const int64_t bc = __ldg(vx.cpu + j), bm = __ldg(vx.mem + j);
        bool keep = rc <= ac - bc && rm <= am - bm;
#pragma unroll
        for (uint32_t k = 0; k < KS_BIND_MAX_RESOURCES; k++) {
            if (k == nreq) break;
            const uint32_t r = rlist >> (4 * k) & 15u;
            keep &= req[r] <= ar[k] - __ldg(fa.vres + (size_t)r * fa.B + j);
        }
        if (keep) { // still fits without evicting b: reprieved
            ac -= bc;
            am -= bm;
#pragma unroll
            for (uint32_t k = 0; k < KS_BIND_MAX_RESOURCES; k++) {
                if (k == nreq) break;
                ar[k] -= __ldg(fa.vres + (size_t)(rlist >> (4 * k) & 15u) * fa.B + j);
            }
            continue;
        }
        if (vcnt == max_victims) return false;
        const int32_t bp = __ldg(vx.prio + j);
        if (vcnt == 0) vmax = bp; // visited in descending priority: the first victim has the highest
        if (out) out[vcnt] = (int32_t)__ldg(vx.idx + j);
        vsum += (int64_t)bp + 2147483648ll;
        vcnt++;
    }
    return true; // at least one victim: with none, the pod would fit every dimension and the node would not be eligible
}

// Candidate scan (ks_fit_preempt): per pod the full-filter feasible count, the unresolvable count, the number of
// candidate nodes and the best candidate's key.  Each cell reads the class's rule word (one coalesced load per node) and,
// where cpu and memory fit on a resolvable node, the free amounts of the pod's requested resources (coalesced as well);
// only eligible cells below min_prio go to fit_preempt_walk.  A warp's pods keep their requests in shared memory and a
// mask of the non-zero ones in registers.  Results go to partials [blockIdx.y][P], merged by k_fit_preempt_emit.
// One pod per warp (FIT_PREEMPT_PODS_PER_WARP): the walks, latency-bound dependent loads, set the time, and with K2p's
// 2-8 pods per warp the walk's R avails took the scan to 210-250 registers, one CTA per SM.  The cell work a warp no
// longer shares across pods is a few shared-memory loads per node.
template <int W>
__global__ void __launch_bounds__(DIRECT_THREADS)
    k_fit_preempt_scan(NodeTable nt, PodView pv, const int32_t* __restrict__ pod_prio, VictimIndex vx, FitPreemptArgs fa,
                       uint32_t max_victims, PreemptPartials part, uint32_t tiles_per_chunk) {
    constexpr int PW = FIT_PREEMPT_PODS_PER_WARP;
    __shared__ int64_t s_req[DIRECT_THREADS / 32][PW][KS_BIND_MAX_RESOURCES];
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int32_t pi[PW];
    uint32_t rmask[PW], rrow[PW]; // non-zero requests; the class's first rule word
    uint64_t bhi[PW], blo[PW];
    uint32_t cnt[PW], ncand[PW], nunres[PW];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t q0 = warp_first_pod<PW>(); // the p0 scan_node_tiles sets
#pragma unroll
    for (int i = 0; i < PW; i++) {
        const uint32_t p = min(q0 + i, pv.P - 1);
        pi[i] = __ldg(pod_prio + p);
        rrow[i] = __ldg(fa.ncls + __ldg(fa.group + p) + 1) * nt.N;
        const int64_t q = lane < fa.R ? __ldg(fa.req + (size_t)p * fa.R + lane) : 0;
        if (lane < KS_BIND_MAX_RESOURCES) s_req[warp][i][lane] = q;
        rmask[i] = __ballot_sync(0xffffffffu, q != 0) & ((1u << KS_BIND_MAX_RESOURCES) - 1u);
        bhi[i] = blo[i] = PREEMPT_NONE;
        cnt[i] = ncand[i] = nunres[i] = 0;
    }
    __syncwarp();

    scan_node_tiles<W, false>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t, int64_t) {
            const int32_t mp = real ? __ldg(vx.min_prio + node) : INT32_MAX; // padding: never a candidate
#pragma unroll
            for (int i = 0; i < PW; i++) {
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const uint32_t word = real ? __ldg(fa.nrules + rrow[i] + node) : 0u;
                const bool resolvable = real && miss == 0 && (word & NR_REASON) == 0;
                bool fit = (rc[i] <= fc) & (rm[i] <= fm);
                if (resolvable && fit) {
#pragma unroll
                    for (uint32_t r = 0; r < KS_BIND_MAX_RESOURCES; r++)
                        if (rmask[i] >> r & 1u) fit &= s_req[warp][i][r] <= __ldg(fa.node_free + (size_t)r * nt.N + node);
                }
                cnt[i] += __popc(__ballot_sync(0xffffffffu, resolvable && fit));
                nunres[i] += __popc(__ballot_sync(0xffffffffu, real && !resolvable));
                if (resolvable && !fit && mp < pi[i]) {
                    int32_t vmax;
                    int64_t vsum;
                    uint32_t vcnt;
                    if (fit_preempt_walk(vx, fa, nt.N, node, pi[i], rc[i], rm[i], fc, fm, s_req[warp][i], rmask[i],
                                         max_victims, vmax, vsum, vcnt, nullptr)) {
                        uint64_t h, l;
                        preempt_key(vmax, vsum, vcnt, node, h, l);
                        ncand[i]++;
                        if (preempt_less(h, l, bhi[i], blo[i])) {
                            bhi[i] = h;
                            blo[i] = l;
                        }
                    }
                }
            }
        },
        [](uint32_t) {});

#pragma unroll
    for (int i = 0; i < PW; i++) {
        uint64_t h = bhi[i], l = blo[i];
        warp_preempt_min(h, l);
        const uint32_t c = __reduce_add_sync(0xffffffffu, ncand[i]);
        const uint32_t p = p0 + i;
        if (lane == 0 && p < pv.P) {
            const uint64_t o = (uint64_t)blockIdx.y * pv.P + p;
            part.hi[o] = h;
            part.lo[o] = l;
            part.cand[o] = c;
            part.cnt[o] = cnt[i];
            fa.unres[o] = nunres[i];
        }
    }
}

// One thread per pod: k_preempt_emit's merge, "already fits => no plan" and row, with fit_preempt_walk for the victims,
// and the unresolvable count.  n_chunks = 0 (no node) gives every pod no plan and 0 unresolvable nodes.
__global__ void __launch_bounds__(256)
    k_fit_preempt_emit(NodeTable nt, PodView pv, const int32_t* __restrict__ pod_prio, VictimIndex vx, FitPreemptArgs fa,
                       uint32_t max_victims, PreemptPartials part, uint32_t n_chunks, ks_preemption* __restrict__ out,
                       int32_t* __restrict__ victims, uint32_t* __restrict__ unres) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pv.P) return;
    uint64_t hi = PREEMPT_NONE, lo = PREEMPT_NONE;
    uint32_t cand = 0, cnt = 0, nu = 0;
    for (uint32_t ch = 0; ch < n_chunks; ch++) {
        const uint64_t o = (uint64_t)ch * pv.P + p;
        cnt += part.cnt[o];
        cand += part.cand[o];
        nu += fa.unres[o];
        if (preempt_less(part.hi[o], part.lo[o], hi, lo)) {
            hi = part.hi[o];
            lo = part.lo[o];
        }
    }
    ks_preemption r;
    r.node_idx = -1;
    r.n_victims = 0;
    r.candidates = cnt ? 0u : cand;
    r.feasible_cnt = cnt;
    r.max_victim_priority = INT32_MIN;
    r.reserved = 0;
    r.victim_priority_sum = 0;
    int32_t* v = victims ? victims + (uint64_t)p * max_victims : nullptr;
    if (cnt == 0 && hi != PREEMPT_NONE) {
        const uint32_t node = (uint32_t)(lo & 0xffffffffffffull);
        const int64_t* req = fa.req + (size_t)p * fa.R;
        uint32_t rmask = 0;
        for (uint32_t k = 0; k < fa.R; k++) rmask |= (req[k] != 0 ? 1u : 0u) << k;
        int32_t vmax;
        int64_t vsum;
        uint32_t vcnt;
        if (fit_preempt_walk(vx, fa, nt.N, node, pod_prio[p], pv.req_cpu[p], pv.req_mem[p], nt.free_cpu[node],
                             nt.free_mem[node], req, rmask, max_victims, vmax, vsum, vcnt, v)) {
            r.node_idx = (int32_t)node;
            r.n_victims = vcnt;
            r.max_victim_priority = vmax;
            r.victim_priority_sum = vsum;
        }
    }
    if (v)
        for (uint32_t j = r.n_victims; j < max_victims; j++) v[j] = -1;
    out[p] = r;
    if (unres) unres[p] = nu;
}

// ------------------------------------------------------------------------------------------------ K2r (ks_drain_check)
// Round r places pod r of every candidate still running (DrainArgs, ks_launch.h).  A candidate's private free f differs
// from free[] only on its overlay nodes, and its own node (plus, with KS_DRAIN_EXCLUDE_CANDIDATES, every candidate's node)
// is no destination.  So the scan reads free[] as K2d does but skips those nodes, through one skip word per (pod, 32
// nodes) built from the node-sorted overlay with a cursor at the start of each tile: the cost is in overlay entries, not
// cells.  The commit step then scores the overlay nodes against f, merges them with the scan's best and records the move.

// Bit (node & 31) of lane (node - tb) / 32's word: nodes tb .. tb + TILE_N - 1 that pod slot p may not take.  xw is this
// lane's word of the excluded-node column; cur is the pod's overlay cursor, advanced past the entries below the tile's
// end.  A failed candidate skips every node.  Called by the whole warp.
__device__ __forceinline__ uint32_t drain_skip_word(const DrainArgs& da, uint32_t p, uint32_t tb, uint32_t xw,
                                                    uint32_t& cur) {
    if (da.failed[p]) return ~0u;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t w = xw;
    const uint32_t cn = (uint32_t)da.cand_node[p];
    if (cn - tb < (uint32_t)TILE_N && lane == (cn - tb) >> 5) w |= 1u << (cn & 31);
    const uint32_t n = da.ov_cnt[p], base = da.pod_base[p];
    while (cur < n) { // warp-uniform: 32 entries per step; the list is sorted, so the entries before the end are a prefix
        const uint32_t k = cur + lane;
        const uint32_t v = k < n ? (uint32_t)da.ov_node[base + k] : 0xffffffffu;
        const uint32_t in = __ballot_sync(0xffffffffu, v < tb + TILE_N);
        for (uint32_t b = in; b; b &= b - 1) {
            const uint32_t nn = __shfl_sync(0xffffffffu, v, __ffs(b) - 1);
            if (nn >= tb && lane == (nn - tb) >> 5) w |= 1u << (nn & 31);
        }
        cur += __popc(in);
        if (in != 0xffffffffu) break;
    }
    return w;
}

template <int W, int POLICY>
// One CTA per SM, as k_select_topk: the skip words and cursors on top of K2d's registers make ptxas spill when held to 128.
__global__ void __launch_bounds__(DIRECT_THREADS, 1)
    k_drain_scan(NodeTable nt, PodView pv, DrainArgs da, PartialView part, uint32_t tiles_per_chunk) {
    constexpr int PW = pods_per_warp(W);
    constexpr bool ALLOC = POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t q0 = warp_first_pod<PW>(); // the p0 scan_node_tiles sets
    bool dead = true; // every pod of this warp failed earlier (or there is none)
#pragma unroll
    for (int i = 0; i < PW; i++)
        if (q0 + i < pv.P && !da.failed[q0 + i]) dead = false;
    if (__syncthreads_and(dead)) return; // the whole CTA: nothing to scan
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int64_t best[PW];
    int32_t bidx[PW];
    uint32_t skip[PW], cur[PW];
#pragma unroll
    for (int i = 0; i < PW; i++) {
        best[i] = INT64_MIN;
        bidx[i] = -1;
        skip[i] = 0;
        cur[i] = 0;
    }

    scan_node_tiles<W, ALLOC>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t g, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t ac, int64_t am) {
            if (g == 0) { // first group of a tile: this tile's skip words
                const uint32_t tb = node - lane;
                const uint32_t xw = da.excl ? __ldg(da.excl + tb / 32 + lane) : 0u;
#pragma unroll
                for (int i = 0; i < PW; i++) skip[i] = drain_skip_word(da, min(p0 + i, pv.P - 1), tb, xw, cur[i]);
            }
            const int64_t key_n = ALLOC ? 0 : leftover_key(fc, fm);
#pragma unroll
            for (int i = 0; i < PW; i++) {
                const bool fit = (rc[i] <= fc) & (rm[i] <= fm);
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const bool off = (__shfl_sync(0xffffffffu, skip[i], g) >> lane) & 1u;
                if (fit && miss == 0 && real && !off) {
                    const int64_t key = ALLOC ? alloc_score<POLICY>(fc, fm, ac, am, rc[i], rm[i]) : key_n;
                    if (key > best[i]) {
                        best[i] = key;
                        bidx[i] = (int32_t)node;
                    }
                }
            }
        },
        [](uint32_t) {});

#pragma unroll
    for (int i = 0; i < PW; i++) {
        int64_t k = best[i];
        int32_t ix = bidx[i];
        warp_argmax(k, ix);
        if (lane == 0 && p0 + i < pv.P) {
            const uint64_t o = (uint64_t)blockIdx.y * pv.P + p0 + i;
            part.key[o] = k;
            part.idx[o] = ix;
        }
    }
}

// One warp per running candidate: the scan's best (chunks merged), the overlay nodes scored against f, the better of the
// two in ks_select's order.  No destination: the candidate fails.  Else the pod's node and score are written, placed
// becomes r + 1, and the move is charged to the overlay - to the node's entry, or a new entry inserted in node order.
template <int W, int POLICY>
__global__ void __launch_bounds__(256)
    k_drain_commit(NodeTable nt, PodView pv, DrainArgs da, PartialView part, uint32_t n_chunks, uint32_t r) {
    constexpr bool ALLOC = POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (p >= pv.P || da.failed[p]) return; // warp-uniform
    const int64_t rc = pv.req_cpu[p], rm = pv.req_mem[p];
    uint64_t sel[W];
#pragma unroll
    for (int w = 0; w < W; w++) sel[w] = pv.sel[(uint64_t)p * W + w];
    int64_t key = INT64_MIN;
    int32_t idx = -1;
    for (uint32_t ch = lane; ch < n_chunks; ch += 32) { // each lane's chunks in ascending order
        const uint64_t o = (uint64_t)ch * pv.P + p;
        merge_partial(key, idx, part.key[o], part.idx[o]);
    }
    const uint32_t n = da.ov_cnt[p], base = da.pod_base[p];
    for (uint32_t k = lane; k < n; k += 32) {
        const int32_t node = da.ov_node[base + k];
        const int64_t fc = da.ov_fc[base + k], fm = da.ov_fm[base + k];
        uint64_t miss = 0;
#pragma unroll
        for (int w = 0; w < W; w++) miss |= sel[w] & ~nt.labels[(uint64_t)w * nt.Npad + node];
        if (rc <= fc && rm <= fm && miss == 0) {
            const int64_t kk = ALLOC ? alloc_score<POLICY>(fc, fm, nt.alloc_cpu[node], nt.alloc_mem[node], rc, rm) : leftover_key(fc, fm);
            if (topk_beats(kk, node, key, idx)) {
                key = kk;
                idx = node;
            }
        }
    }
    warp_argmax(key, idx);
    if (idx < 0) {
        if (lane == 0) da.failed[p] = 1;
        return;
    }
    const uint32_t pod = da.pod_base[p] + r;
    if (lane == 0) {
        da.out_idx[pod] = idx;
        da.out_score[pod] = ALLOC ? key : leftover_score(key, rc, rm);
        da.placed[da.cand_id[p]] = r + 1;
    }
    uint32_t pos = 0; // entries below idx
    bool found = false;
    for (uint32_t k0 = 0; k0 < n; k0 += 32) {
        const uint32_t k = k0 + lane;
        const int32_t v = k < n ? da.ov_node[base + k] : INT32_MAX;
        pos += __popc(__ballot_sync(0xffffffffu, v < idx));
        found |= __any_sync(0xffffffffu, v == idx);
    }
    if (found) {
        if (lane == 0) {
            da.ov_fc[base + pos] -= rc;
            da.ov_fm[base + pos] -= rm;
        }
        return;
    }
    for (uint32_t top = n; top > pos; top = top > pos + 32 ? top - 32 : pos) { // shift [pos, n) up one, top chunk first
        const int64_t k = (int64_t)top - 1 - lane;
        const bool mv = k >= (int64_t)pos;
        int32_t vn = 0;
        int64_t vc = 0, vm = 0;
        if (mv) {
            vn = da.ov_node[base + k];
            vc = da.ov_fc[base + k];
            vm = da.ov_fm[base + k];
        }
        __syncwarp();
        if (mv) {
            da.ov_node[base + k + 1] = vn;
            da.ov_fc[base + k + 1] = vc;
            da.ov_fm[base + k + 1] = vm;
        }
        __syncwarp();
    }
    if (lane == 0) {
        da.ov_node[base + pos] = idx;
        da.ov_fc[base + pos] = nt.free_cpu[idx] - rc;
        da.ov_fm[base + pos] = nt.free_mem[idx] - rm;
        da.ov_cnt[p] = n + 1;
    }
}

// ------------------------------------------------------------------------------------------------ K2u (ks_fit_drain_check)
// K2r under the full filter (include/ksched.h, ks_fit_drain_check).  A destination that passes cpu, memory and the
// selector also needs its class's rule word (one coalesced load per node) and, for each resource the pod requests, its
// free amount: node_free in the scan, the overlay's ov_fr column in the commit.  Scores stay the policy's over f.
// COUNT: the refusal pass after the last round, over the stopping pods of the stopped candidates (fa.stopped), whose
// overlays are frozen since their stop.  Each destination lands in one of four words by the first filter it fails; the
// scan counts the nodes off the overlay, the warp of node chunk 0 then the overlay nodes, so the words sum to the
// destination count.  One pod per warp (FIT_DRAIN_PODS_PER_WARP): with K2d's 2-8 the scan took 236-255 registers at
// W = 1 and 2, spilled in the refusal pass, and the c3 sweep ran 31% slower (DESIGN.md 5u).
template <int W, int POLICY, bool COUNT>
__global__ void __launch_bounds__(DIRECT_THREADS, 1)
    k_fit_drain_scan(NodeTable nt, PodView pv, DrainArgs da, FitDrainArgs fa, PartialView part, uint32_t tiles_per_chunk) {
    constexpr int PW = FIT_DRAIN_PODS_PER_WARP;
    constexpr bool ALLOC = !COUNT && POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    __shared__ int64_t s_req[DIRECT_THREADS / 32][PW][KS_BIND_MAX_RESOURCES];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t q0 = warp_first_pod<PW>(); // the p0 scan_node_tiles sets
    bool dead = true; // every pod of this warp is done (or there is none)
#pragma unroll
    for (int i = 0; i < PW; i++)
        if (q0 + i < pv.P && (COUNT ? fa.stopped[q0 + i] != 0 : !da.failed[q0 + i])) dead = false;
    if (__syncthreads_and(dead)) return; // the whole CTA: nothing to scan
    int64_t rc[PW], rm[PW];
    uint64_t sel[PW][W];
    uint32_t p0;
    int64_t best[PW];
    int32_t bidx[PW];
    uint32_t skip[PW], cur[PW];
    uint32_t rmask[PW], rrow[PW]; // non-zero requests; the class's first rule word
    uint32_t nref[PW][4];         // COUNT: the four words
#pragma unroll
    for (int i = 0; i < PW; i++) {
        const uint32_t p = min(q0 + i, pv.P - 1);
        // COUNT: the commit wrote a slot's stop record only if its candidate stopped; any other slot reads as group -1
        // with no request, so that its leftover bytes index nothing (its counts are never written)
        const bool live = !COUNT || fa.stopped[p] != 0;
        rrow[i] = __ldg(fa.ncls + (live ? __ldg(fa.group + p) : -1) + 1) * nt.N;
        const int64_t q = live && lane < fa.R ? __ldg(fa.req + (size_t)p * fa.R + lane) : 0;
        if (lane < KS_BIND_MAX_RESOURCES) s_req[warp][i][lane] = q;
        rmask[i] = __ballot_sync(0xffffffffu, q != 0) & ((1u << KS_BIND_MAX_RESOURCES) - 1u);
        best[i] = INT64_MIN;
        bidx[i] = -1;
        skip[i] = 0;
        cur[i] = 0;
        nref[i][0] = nref[i][1] = nref[i][2] = nref[i][3] = 0;
    }
    __syncwarp();

    scan_node_tiles<W, ALLOC>(
        nt, tiles_per_chunk, pv, p0, rc, rm, sel,
        [&](uint32_t g, uint32_t node, bool real, int64_t fc, int64_t fm, const uint64_t(&lab)[W], int64_t ac, int64_t am) {
            if (g == 0) { // first group of a tile: this tile's skip words
                const uint32_t tb = node - lane;
                const uint32_t xw = da.excl ? __ldg(da.excl + tb / 32 + lane) : 0u;
#pragma unroll
                for (int i = 0; i < PW; i++) skip[i] = drain_skip_word(da, min(p0 + i, pv.P - 1), tb, xw, cur[i]);
            }
#pragma unroll
            for (int i = 0; i < PW; i++) {
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~lab[w];
                const bool off = (__shfl_sync(0xffffffffu, skip[i], g) >> lane) & 1u;
                const bool dest = real && !off;
                const bool pass = dest && (rc[i] <= fc) && (rm[i] <= fm) && miss == 0;
                uint32_t word = 0;
                bool fit_r = true;
                if (pass) {
                    word = __ldg(fa.nrules + rrow[i] + node) & NR_REASON;
#pragma unroll
                    for (uint32_t r = 0; r < KS_BIND_MAX_RESOURCES; r++)
                        if (rmask[i] >> r & 1u) fit_r &= s_req[warp][i][r] <= __ldg(fa.node_free + (size_t)r * nt.N + node);
                }
                if (COUNT) {
                    nref[i][0] += __popc(__ballot_sync(0xffffffffu, dest && !pass));
                    nref[i][1] += __popc(__ballot_sync(0xffffffffu, pass && !fit_r));
                    nref[i][2] += __popc(__ballot_sync(0xffffffffu, pass && fit_r && word == NR_TAINT));
                    nref[i][3] += __popc(__ballot_sync(0xffffffffu, pass && fit_r && word == NR_AFFINITY));
                } else if (pass && fit_r && word == 0) {
                    const int64_t key = ALLOC ? alloc_score<POLICY>(fc, fm, ac, am, rc[i], rm[i]) : leftover_key(fc, fm);
                    if (key > best[i]) {
                        best[i] = key;
                        bidx[i] = (int32_t)node;
                    }
                }
            }
        },
        [](uint32_t) {});

#pragma unroll
    for (int i = 0; i < PW; i++) {
        const uint32_t p = p0 + i;
        if (!COUNT) {
            int64_t k = best[i];
            int32_t ix = bidx[i];
            warp_argmax(k, ix);
            if (lane == 0 && p < pv.P) {
                const uint64_t o = (uint64_t)blockIdx.y * pv.P + p;
                part.key[o] = k;
                part.idx[o] = ix;
            }
            continue;
        }
        if (p >= pv.P || !fa.stopped[p]) continue; // warp-uniform
        if (blockIdx.y == 0) { // the overlay nodes, against f and f_r
            const uint32_t n = da.ov_cnt[p], base = da.pod_base[p];
            for (uint32_t k0 = 0; k0 < n; k0 += 32) {
                const uint32_t k = k0 + lane;
                const bool v = k < n;
                const int32_t node = v ? da.ov_node[base + k] : 0;
                uint64_t miss = 0;
#pragma unroll
                for (int w = 0; w < W; w++) miss |= sel[i][w] & ~nt.labels[(uint64_t)w * nt.Npad + node];
                const bool pass = v && rc[i] <= da.ov_fc[base + k] && rm[i] <= da.ov_fm[base + k] && miss == 0;
                uint32_t word = 0;
                bool fit_r = true;
                if (pass) {
                    word = fa.nrules[rrow[i] + node] & NR_REASON;
                    for (uint32_t r = 0; r < fa.R; r++)
                        if (rmask[i] >> r & 1u) fit_r &= s_req[warp][i][r] <= fa.ov_fr[(size_t)r * fa.P + base + k];
                }
                nref[i][0] += __popc(__ballot_sync(0xffffffffu, v && !pass));
                nref[i][1] += __popc(__ballot_sync(0xffffffffu, pass && !fit_r));
                nref[i][2] += __popc(__ballot_sync(0xffffffffu, pass && fit_r && word == NR_TAINT));
                nref[i][3] += __popc(__ballot_sync(0xffffffffu, pass && fit_r && word == NR_AFFINITY));
            }
        }
        const uint32_t c = lane == 0 ? nref[i][0] : lane == 1 ? nref[i][1] : lane == 2 ? nref[i][2] : nref[i][3];
        if (lane < 4 && c) atomicAdd(fa.refused + 4 * (size_t)da.cand_id[p] + lane, c); // integer adds: any order
    }
}

// k_drain_commit with the full filter: an overlay node also needs the class's rule word to pass and each requested
// resource to fit its ov_fr column; the move charges f_r along with f, and an insert shifts the R columns with the
// rest.  A candidate that stops leaves its stopping pod in the stop arrays when fa.stop_cpu is set.
template <int W, int POLICY>
__global__ void __launch_bounds__(256, 1)
    k_fit_drain_commit(NodeTable nt, PodView pv, DrainArgs da, FitDrainArgs fa, PartialView part, uint32_t n_chunks,
                       uint32_t r) {
    constexpr bool ALLOC = POLICY != KS_SCORE_LEFTOVER; // scored from the allocatables
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (p >= pv.P || da.failed[p]) return; // warp-uniform
    const int64_t rc = pv.req_cpu[p], rm = pv.req_mem[p];
    const uint64_t* sel = pv.sel + (uint64_t)p * W; // read where it is used: nothing but the loop state lives across
    const uint32_t R = fa.R;                        // alloc_score's int64 divisions
    const int64_t* req = fa.req + (size_t)p * R;
    const uint32_t rmask = __ballot_sync(0xffffffffu, lane < R && req[lane] != 0); // the requested resources
    const uint32_t rrow = fa.ncls[fa.group[p] + 1] * nt.N;
    int64_t key = INT64_MIN;
    int32_t idx = -1;
    for (uint32_t ch = lane; ch < n_chunks; ch += 32) { // each lane's chunks in ascending order
        const uint64_t o = (uint64_t)ch * pv.P + p;
        merge_partial(key, idx, part.key[o], part.idx[o]);
    }
    const uint32_t n = da.ov_cnt[p], base = da.pod_base[p];
#pragma unroll 1
    for (uint32_t k0 = 0; k0 < n; k0 += 32) {
        const uint32_t k = k0 + lane;
        const int32_t node = k < n ? da.ov_node[base + k] : 0;
        const int64_t fc = k < n ? da.ov_fc[base + k] : 0, fm = k < n ? da.ov_fm[base + k] : 0;
        uint64_t miss = 0;
#pragma unroll
        for (int w = 0; w < W; w++) miss |= sel[w] & ~nt.labels[(uint64_t)w * nt.Npad + node];
        bool ok = k < n && rc <= fc && rm <= fm && miss == 0 && (fa.nrules[rrow + node] & NR_REASON) == 0;
        for (uint32_t m = rmask; m; m &= m - 1) { // a zero request always fits
            const uint32_t j = __ffs(m) - 1;
            if (ok) ok = req[j] <= fa.ov_fr[(size_t)j * fa.P + base + k];
        }
        if (ok) {
            const int64_t kk = ALLOC ? alloc_score<POLICY>(fc, fm, nt.alloc_cpu[node], nt.alloc_mem[node], rc, rm) : leftover_key(fc, fm);
            if (topk_beats(kk, node, key, idx)) {
                key = kk;
                idx = node;
            }
        }
    }
    warp_argmax(key, idx);
    const int64_t rq = lane < R ? req[lane] : 0; // lane j: the request of resource j
    if (idx < 0) {
        if (fa.stop_cpu) { // the stopping pod, for the refusal pass
            if (lane == 0) {
                fa.stop_cpu[p] = rc;
                fa.stop_mem[p] = rm;
                fa.stop_grp[p] = fa.group[p];
            }
            if (lane < W) fa.stop_sel[(uint64_t)p * W + lane] = pv.sel[(uint64_t)p * W + lane];
            if (lane < R) fa.stop_req[(size_t)p * R + lane] = rq;
        }
        if (lane == 0) da.failed[p] = 1;
        return;
    }
    const uint32_t pod = da.pod_base[p] + r;
    if (lane == 0) {
        da.out_idx[pod] = idx;
        da.out_score[pod] = ALLOC ? key : leftover_score(key, rc, rm);
        da.placed[da.cand_id[p]] = r + 1;
    }
    uint32_t pos = 0; // entries below idx
    bool found = false;
    for (uint32_t k0 = 0; k0 < n; k0 += 32) {
        const uint32_t k = k0 + lane;
        const int32_t v = k < n ? da.ov_node[base + k] : INT32_MAX;
        pos += __popc(__ballot_sync(0xffffffffu, v < idx));
        found |= __any_sync(0xffffffffu, v == idx);
    }
    if (found) {
        if (lane == 0) {
            da.ov_fc[base + pos] -= rc;
            da.ov_fm[base + pos] -= rm;
        }
        if (lane < R) fa.ov_fr[(size_t)lane * fa.P + base + pos] -= rq;
        return;
    }
    for (uint32_t top = n; top > pos; top = top > pos + 32 ? top - 32 : pos) { // shift [pos, n) up one, top chunk first
        const int64_t k = (int64_t)top - 1 - lane;
        const bool mv = k >= (int64_t)pos;
        int32_t vn = 0;
        int64_t vc = 0, vm = 0;
        if (mv) {
            vn = da.ov_node[base + k];
            vc = da.ov_fc[base + k];
            vm = da.ov_fm[base + k];
        }
        __syncwarp();
        if (mv) {
            da.ov_node[base + k + 1] = vn;
            da.ov_fc[base + k + 1] = vc;
            da.ov_fm[base + k + 1] = vm;
        }
        __syncwarp();
#pragma unroll 1
        for (uint32_t j = 0; j < R; j++) { // the R columns, one at a time
            int64_t* col = fa.ov_fr + (size_t)j * fa.P + base;
            const int64_t v = mv ? col[k] : 0;
            __syncwarp();
            if (mv) col[k + 1] = v;
            __syncwarp();
        }
    }
    if (lane == 0) {
        da.ov_node[base + pos] = idx;
        da.ov_fc[base + pos] = nt.free_cpu[idx] - rc;
        da.ov_fm[base + pos] = nt.free_mem[idx] - rm;
        da.ov_cnt[p] = n + 1;
    }
    if (lane < R)
        fa.ov_fr[(size_t)lane * fa.P + base + pos] = fa.node_free[(size_t)lane * nt.N + idx] - rq;
}

// ---- the victim index, built per call: a stable LSD radix sort of (node << 32 | priority + 2^31) keys over the bound
// list fed in descending bound index, then segment offsets, prefix sums and per-node minimum priorities.
constexpr uint32_t RADIX_TILE = 2048; // keys per CTA of a radix pass (256 threads x 8 rounds)

__global__ void __launch_bounds__(256)
    k_victim_keys(const int32_t* __restrict__ bnode, const int32_t* __restrict__ bprio, uint64_t* __restrict__ key,
                  uint32_t* __restrict__ val, uint64_t B) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = B - 1 - i; // reversed: the stable sort leaves ties in descending bound index
        key[i] = ((uint64_t)(uint32_t)bnode[b] << 32) | ((uint32_t)bprio[b] ^ 0x80000000u);
        val[i] = (uint32_t)b;
    }
}

// per CTA tile: counts of each 8-bit digit, stored digit-major (hist[d * nblk + tile]) so that one exclusive scan over
// the whole array gives every (digit, tile) its first output position
__global__ void __launch_bounds__(256)
    k_radix_hist(const uint64_t* __restrict__ key, uint64_t B, uint32_t shift, uint32_t* __restrict__ hist, uint32_t nblk) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * RADIX_TILE;
    for (uint32_t j = threadIdx.x; j < RADIX_TILE; j += 256)
        if (base + j < B) atomicAdd(&h[(uint32_t)(key[base + j] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(uint64_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// one CTA: exclusive scan of n counts in place (each thread scans a contiguous run, then the run totals are scanned)
__global__ void __launch_bounds__(1024) k_radix_scan(uint32_t* __restrict__ a, uint32_t n) {
    __shared__ uint32_t tot[1024];
    const uint32_t per = (n + 1023) / 1024, b = threadIdx.x * per, e = min(b + per, n);
    uint32_t s = 0;
    for (uint32_t i = b; i < e; i++) s += a[i];
    tot[threadIdx.x] = s;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) { // Hillis-Steele over the run totals
        const uint32_t v = threadIdx.x >= off ? tot[threadIdx.x - off] : 0;
        __syncthreads();
        tot[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = tot[threadIdx.x] - s;
    for (uint32_t i = b; i < e; i++) {
        const uint32_t x = a[i];
        a[i] = run;
        run += x;
    }
}

// Stable scatter of one radix pass.  A CTA takes its tile in rounds of 256 keys in order; within a round, warps hold
// consecutive keys and peers of a digit are ranked by lane (match_any), so every key lands after all earlier keys of its
// digit: the pass is stable.
__global__ void __launch_bounds__(256)
    k_radix_scatter(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin, uint64_t* __restrict__ kout,
                    uint32_t* __restrict__ vout, uint64_t B, uint32_t shift, const uint32_t* __restrict__ hist,
                    uint32_t nblk) {
    __shared__ uint32_t base[256];
    __shared__ uint32_t wcnt[8][256];
    const uint32_t t = threadIdx.x, lane = t & 31, w = t >> 5;
    base[t] = hist[(uint64_t)t * nblk + blockIdx.x];
#pragma unroll
    for (int q = 0; q < 8; q++) wcnt[q][t] = 0;
    __syncthreads();
    const uint64_t tile = (uint64_t)blockIdx.x * RADIX_TILE;
    for (uint32_t r = 0; r < RADIX_TILE / 256; r++) {
        const uint64_t i = tile + r * 256 + t;
        const bool valid = i < B;
        const uint64_t k = valid ? kin[i] : 0;
        const uint32_t v = valid ? vin[i] : 0;
        const uint32_t d = (uint32_t)(k >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xffffffffu, valid ? d : 256u);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) wcnt[w][d] = __popc(peers);
        __syncthreads();
        if (valid) {
            uint32_t pos = base[d] + rank;
            for (uint32_t q = 0; q < w; q++) pos += wcnt[q][d];
            kout[pos] = k;
            vout[pos] = v;
        }
        __syncthreads();
        uint32_t add = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            add += wcnt[q][t];
            wcnt[q][t] = 0;
        }
        base[t] += add;
        __syncthreads();
    }
}

// sorted arrays: priority (from the key), requests gathered by bound index
__global__ void __launch_bounds__(256)
    k_victim_gather(const uint64_t* __restrict__ key, const uint32_t* __restrict__ val, const int64_t* __restrict__ bcpu,
                    const int64_t* __restrict__ bmem, int32_t* __restrict__ prio, int64_t* __restrict__ cpu,
                    int64_t* __restrict__ mem, uint64_t B) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < B; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = val[j];
        prio[j] = (int32_t)((uint32_t)key[j] ^ 0x80000000u);
        cpu[j] = bcpu[b];
        mem[j] = bmem[b];
    }
}

// off[n] = first sorted position of node n (n = N gives B): a binary search over the sorted keys
__global__ void __launch_bounds__(256)
    k_victim_offsets(const uint64_t* __restrict__ key, uint64_t B, uint32_t N, uint32_t* __restrict__ off) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n > N) return;
    const uint64_t want = (uint64_t)n << 32;
    uint64_t lo = 0, hi = B;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (key[mid] < want) lo = mid + 1;
        else hi = mid;
    }
    off[n] = (uint32_t)lo;
}

// one warp per node: inclusive prefix sums of the segment's requests, 32 at a time, and its lowest priority
__global__ void __launch_bounds__(256)
    k_victim_prefix(const uint32_t* __restrict__ off, const int32_t* __restrict__ prio, const int64_t* __restrict__ cpu,
                    const int64_t* __restrict__ mem, int64_t* __restrict__ pre_cpu, int64_t* __restrict__ pre_mem,
                    int32_t* __restrict__ min_prio, uint32_t N) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return; // warp-uniform
    const uint32_t s0 = off[n], s1 = off[n + 1];
    int64_t carry_c = 0, carry_m = 0;
    for (uint32_t j0 = s0; j0 < s1; j0 += 32) {
        const uint32_t j = j0 + lane;
        int64_t c = j < s1 ? cpu[j] : 0, m = j < s1 ? mem[j] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t uc = __shfl_up_sync(0xffffffffu, c, d), um = __shfl_up_sync(0xffffffffu, m, d);
            if (lane >= (uint32_t)d) {
                c += uc;
                m += um;
            }
        }
        if (j < s1) {
            pre_cpu[j] = carry_c + c;
            pre_mem[j] = carry_m + m;
        }
        carry_c += __shfl_sync(0xffffffffu, c, 31);
        carry_m += __shfl_sync(0xffffffffu, m, 31);
    }
    if (lane == 0) min_prio[n] = s1 > s0 ? prio[s0] : INT32_MAX;
}

// ks_fit_preempt's request columns: vres[r * B + j] = breq[idx[j] * R + r], gathered through the sorted bound indices
__global__ void __launch_bounds__(256)
    k_victim_gather_res(const uint32_t* __restrict__ idx, const int64_t* __restrict__ breq, int64_t* __restrict__ vres,
                        uint32_t B, uint32_t R) {
    const uint64_t total = (uint64_t)B * R;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(i / B), j = (uint32_t)(i % B);
        vres[i] = breq[(uint64_t)idx[j] * R + r];
    }
}

// one warp per (node, column blockIdx.y): inclusive prefix sums of the column within the node's segment, as
// k_victim_prefix sums cpu and memory
__global__ void __launch_bounds__(256)
    k_victim_prefix_res(const uint32_t* __restrict__ off, const int64_t* __restrict__ vres, int64_t* __restrict__ vpre,
                        uint32_t N, uint32_t B) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return; // warp-uniform
    const int64_t* col = vres + (size_t)blockIdx.y * B;
    int64_t* pre = vpre + (size_t)blockIdx.y * B;
    const uint32_t s0 = off[n], s1 = off[n + 1];
    int64_t carry = 0;
    for (uint32_t j0 = s0; j0 < s1; j0 += 32) {
        const uint32_t j = j0 + lane;
        int64_t c = j < s1 ? col[j] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t u = __shfl_up_sync(0xffffffffu, c, d);
            if (lane >= (uint32_t)d) c += u;
        }
        if (j < s1) pre[j] = carry + c;
        carry += __shfl_sync(0xffffffffu, c, 31);
    }
}

// scratch layout: the upload, two key/value buffers of the sort, the digit counts, then the index itself
struct VictimLayout {
    size_t node, cpu, mem, prio, key[2], val[2], hist, s_prio, s_cpu, s_mem, pre_cpu, pre_mem, off, min_prio, total;
    uint32_t nblk;
};
static VictimLayout victim_layout(uint64_t B, uint32_t N) {
    VictimLayout L;
    BlockLayout b; // every array 256-byte aligned
    L.nblk = (uint32_t)((B + RADIX_TILE - 1) / RADIX_TILE);
    L.node = b.take<int32_t>(B, 256);
    L.cpu = b.take<int64_t>(B, 256);
    L.mem = b.take<int64_t>(B, 256);
    L.prio = b.take<int32_t>(B, 256);
    L.key[0] = b.take<uint64_t>(B, 256);
    L.key[1] = b.take<uint64_t>(B, 256);
    L.val[0] = b.take<uint32_t>(B, 256);
    L.val[1] = b.take<uint32_t>(B, 256);
    L.hist = b.take<uint32_t>((size_t)256 * L.nblk, 256);
    L.s_prio = b.take<int32_t>(B, 256);
    L.s_cpu = b.take<int64_t>(B, 256);
    L.s_mem = b.take<int64_t>(B, 256);
    L.pre_cpu = b.take<int64_t>(B, 256);
    L.pre_mem = b.take<int64_t>(B, 256);
    L.off = b.take<uint32_t>((size_t)N + 1, 256);
    L.min_prio = b.take<int32_t>(N, 256);
    L.total = b.size;
    return L;
}

size_t victim_index_bytes(uint64_t B, uint32_t N) { return victim_layout(B, N).total; }

BoundUpload victim_index_inputs(void* scratch, uint64_t B, uint32_t N) {
    const VictimLayout L = victim_layout(B, N);
    return BoundUpload{at<int32_t>(scratch, L.node), at<int64_t>(scratch, L.cpu), at<int64_t>(scratch, L.mem),
                       at<int32_t>(scratch, L.prio)};
}

cudaError_t build_victim_index(void* scratch, uint64_t B, uint32_t N, VictimIndex* vx, cudaStream_t st) {
    const VictimLayout L = victim_layout(B, N);
    void* s = scratch;
    uint64_t* key[2] = {at<uint64_t>(s, L.key[0]), at<uint64_t>(s, L.key[1])};
    uint32_t* val[2] = {at<uint32_t>(s, L.val[0]), at<uint32_t>(s, L.val[1])};
    int cur = 0;
    const uint32_t grid_b = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(4096, (B + 255) / 256));
    cudaError_t e;
    if (B) {
        k_victim_keys<<<grid_b, 256, 0, st>>>(at<int32_t>(s, L.node), at<int32_t>(s, L.prio), key[0], val[0], B);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        // priority bits [0, 32), then as many node bits as N needs
        const uint32_t node_bits = N > 1 ? 32u - (uint32_t)__builtin_clz(N - 1) : 0u;
        for (uint32_t shift = 0; shift < 32 + node_bits; shift += 8) {
            uint32_t* hist = at<uint32_t>(s, L.hist);
            k_radix_hist<<<L.nblk, 256, 0, st>>>(key[cur], B, shift, hist, L.nblk);
            k_radix_scan<<<1, 1024, 0, st>>>(hist, 256 * L.nblk);
            k_radix_scatter<<<L.nblk, 256, 0, st>>>(key[cur], val[cur], key[cur ^ 1], val[cur ^ 1], B, shift, hist, L.nblk);
            g_launches += 3;
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            cur ^= 1;
        }
        k_victim_gather<<<grid_b, 256, 0, st>>>(key[cur], val[cur], at<int64_t>(s, L.cpu), at<int64_t>(s, L.mem),
                                                at<int32_t>(s, L.s_prio), at<int64_t>(s, L.s_cpu),
                                                at<int64_t>(s, L.s_mem), B);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    k_victim_offsets<<<(N + 1 + 255) / 256, 256, 0, st>>>(key[cur], B, N, at<uint32_t>(s, L.off));
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (N) {
        k_victim_prefix<<<(N + 7) / 8, 256, 0, st>>>(at<uint32_t>(s, L.off), at<int32_t>(s, L.s_prio),
                                                     at<int64_t>(s, L.s_cpu), at<int64_t>(s, L.s_mem),
                                                     at<int64_t>(s, L.pre_cpu), at<int64_t>(s, L.pre_mem),
                                                     at<int32_t>(s, L.min_prio), N);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    vx->off = at<uint32_t>(s, L.off);
    vx->min_prio = at<int32_t>(s, L.min_prio);
    vx->prio = at<int32_t>(s, L.s_prio);
    vx->cpu = at<int64_t>(s, L.s_cpu);
    vx->mem = at<int64_t>(s, L.s_mem);
    vx->pre_cpu = at<int64_t>(s, L.pre_cpu);
    vx->pre_mem = at<int64_t>(s, L.pre_mem);
    vx->idx = val[cur];
    return cudaSuccess;
}

cudaError_t build_fit_victim_index(const VictimIndex& vx, const int64_t* breq, const FitPreemptArgs& fa, uint32_t N,
                                   cudaStream_t st) {
    if (fa.R == 0 || fa.B == 0 || N == 0) return cudaSuccess;
    const uint64_t total = (uint64_t)fa.B * fa.R;
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(4096, (total + 255) / 256));
    k_victim_gather_res<<<grid, 256, 0, st>>>(vx.idx, breq, const_cast<int64_t*>(fa.vres), fa.B, fa.R);
    k_victim_prefix_res<<<dim3((N + 7) / 8, fa.R), 256, 0, st>>>(vx.off, fa.vres, const_cast<int64_t*>(fa.vpre), N,
                                                                 fa.B);
    g_launches += 2;
    return cudaGetLastError();
}

// node chunks across gridDim.y when the pods alone give fewer than two CTAs per SM
static DirectGrid direct_grid_ppw(uint32_t ppw, uint32_t P, uint32_t Npad, int sms) {
    const uint32_t pods_per_cta = (DIRECT_THREADS / 32) * ppw;
    const uint32_t n_tiles = Npad / TILE_N;
    const uint32_t want_ctas = 2u * (uint32_t)sms;
    DirectGrid g;
    g.pod_ctas = (P + pods_per_cta - 1) / pods_per_cta;
    g.n_chunks = 1;
    if (g.pod_ctas < want_ctas) g.n_chunks = std::min<uint32_t>(n_tiles, (want_ctas + g.pod_ctas - 1) / g.pod_ctas);
    g.tiles_per_chunk = (n_tiles + g.n_chunks - 1) / g.n_chunks;
    g.n_chunks = (n_tiles + g.tiles_per_chunk - 1) / g.tiles_per_chunk;
    return g;
}

DirectGrid direct_grid(uint32_t W, uint32_t P, uint32_t Npad, int sms) { return direct_grid_ppw(pods_per_warp(W), P, Npad, sms); }

DirectGrid fit_preempt_grid(uint32_t P, uint32_t Npad, int sms) {
    return direct_grid_ppw(FIT_PREEMPT_PODS_PER_WARP, P, Npad, sms);
}

DirectGrid fit_drain_grid(uint32_t P, uint32_t Npad, int sms) { return direct_grid_ppw(FIT_DRAIN_PODS_PER_WARP, P, Npad, sms); }

// opt-in shared memory sizes of every K2d / K2e kernel on the current device (must not run inside a stream capture)
cudaError_t prepare_direct() {
    cudaError_t e = cudaSuccess;
    auto opt_in = [&e](auto kern, uint32_t bytes) {
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    };
    for (uint32_t W : {1u, 2u, 4u, 8u})
        with_label_width(W, [&](auto w) {
            constexpr int W_ = decltype(w)::value;
            opt_in(k_explain_counts<W_>, tile_smem_bytes<W_, false>());
            opt_in(k_preempt_scan<W_>, tile_smem_bytes<W_, false>());
            opt_in(k_fit_preempt_scan<W_>, tile_smem_bytes<W_, false>());
            opt_in(k_fit_drain_scan<W_, KS_SCORE_LEFTOVER, true>, tile_smem_bytes<W_, false>());
            for (int policy : {KS_SCORE_LEFTOVER, KS_SCORE_LEAST_ALLOCATED, KS_SCORE_MOST_ALLOCATED, KS_SCORE_LEAST_BALANCED})
                with_policy(policy, [&](auto pol) {
                    constexpr int POL = decltype(pol)::value;
                    constexpr uint32_t SMEM = tile_smem_bytes<W_, POL != KS_SCORE_LEFTOVER>();
                    opt_in(k_select_direct<W_, POL, true>, SMEM);
                    opt_in(k_select_direct<W_, POL, false>, SMEM);
                    opt_in(k_select_topk<W_, POL>, SMEM);
                    opt_in(k_drain_scan<W_, POL>, SMEM);
                    opt_in(k_fit_drain_scan<W_, POL, false>, SMEM);
                    return e;
                });
            return e;
        });
    return e;
}

template <int W, int POLICY, bool EMIT>
static cudaError_t launch_direct_t(const SelectLaunch& L, const PartialView& part, const DirectGrid& g) {
    constexpr uint32_t SMEM = tile_smem_bytes<W, POLICY != KS_SCORE_LEFTOVER>();
    k_select_direct<W, POLICY, EMIT><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, SMEM, L.stream>>>(
        L.nt, L.pv, L.ov, part, g.tiles_per_chunk);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || g.n_chunks == 1) return e;
    k_select_combine<POLICY><<<(L.pv.P + 255) / 256, 256, 0, L.stream>>>(L.pv, L.ov, part, g.n_chunks);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_select_direct(const SelectLaunch& L, const PartialView& part, const DirectGrid& g) {
    return with_label_width(L.nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        return with_policy(L.policy, [&](auto pol) {
            constexpr int POL = decltype(pol)::value;
            return L.ov.mask ? launch_direct_t<W, POL, true>(L, part, g) : launch_direct_t<W, POL, false>(L, part, g);
        });
    });
}

cudaError_t launch_explain_counts(const NodeTable& nt, const PodView& pv, uint32_t* out, int sms, cudaStream_t st) {
    if (pv.P == 0 || nt.Npad == 0) return cudaSuccess;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        const DirectGrid g = direct_grid(W, pv.P, nt.Npad, sms);
        if (g.n_chunks > 1) {
            const cudaError_t e = cudaMemsetAsync(out, 0, (size_t)pv.P * 16, st);
            if (e != cudaSuccess) return e;
        }
        k_explain_counts<W><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, tile_smem_bytes<W, false>(), st>>>(
            nt, pv, out, g.tiles_per_chunk);
        g_launches++;
        return cudaGetLastError();
    });
}

template <int W, int POLICY>
static cudaError_t launch_topk_t(const NodeTable& nt, const PodView& pv, uint32_t k, const OutView& ov,
                                 const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    constexpr uint32_t SMEM = tile_smem_bytes<W, POLICY != KS_SCORE_LEFTOVER>();
    k_select_topk<W, POLICY><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, SMEM, st>>>(nt, pv, ov, part, k,
                                                                                          g.tiles_per_chunk);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || g.n_chunks == 1) return e;
    k_topk_combine<POLICY><<<(pv.P + 7) / 8, 256, 0, st>>>(pv, ov, part, g.n_chunks, k);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_select_topk(const NodeTable& nt, const PodView& pv, int policy, uint32_t k, const OutView& ov,
                               const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        return with_policy(policy, [&](auto pol) {
            return launch_topk_t<W, decltype(pol)::value>(nt, pv, k, ov, part, g, st);
        });
    });
}

cudaError_t launch_preempt(const NodeTable& nt, const PodView& pv, const int32_t* pod_prio, const VictimIndex& vx,
                           uint32_t max_victims, const PreemptPartials& part, const DirectGrid& g, ks_preemption* out,
                           int32_t* victims, cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    uint32_t n_chunks = 0;
    if (nt.N > 0) {
        const cudaError_t e = with_label_width(nt.W, [&](auto w) {
            constexpr int W = decltype(w)::value;
            k_preempt_scan<W><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, tile_smem_bytes<W, false>(), st>>>(
                nt, pv, pod_prio, vx, max_victims, part, g.tiles_per_chunk);
            g_launches++;
            return cudaGetLastError();
        });
        if (e != cudaSuccess) return e;
        n_chunks = g.n_chunks;
    }
    k_preempt_emit<<<(pv.P + 255) / 256, 256, 0, st>>>(nt, pv, pod_prio, vx, max_victims, part, n_chunks, out, victims);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_fit_preempt(const NodeTable& nt, const PodView& pv, const int32_t* pod_prio, const VictimIndex& vx,
                               const FitPreemptArgs& fa, uint32_t max_victims, const PreemptPartials& part,
                               const DirectGrid& g, ks_preemption* out, int32_t* victims, uint32_t* unres,
                               cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    uint32_t n_chunks = 0;
    if (nt.N > 0) {
        const cudaError_t e = with_label_width(nt.W, [&](auto w) {
            constexpr int W = decltype(w)::value;
            k_fit_preempt_scan<W><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, tile_smem_bytes<W, false>(), st>>>(
                nt, pv, pod_prio, vx, fa, max_victims, part, g.tiles_per_chunk);
            g_launches++;
            return cudaGetLastError();
        });
        if (e != cudaSuccess) return e;
        n_chunks = g.n_chunks;
    }
    k_fit_preempt_emit<<<(pv.P + 255) / 256, 256, 0, st>>>(nt, pv, pod_prio, vx, fa, max_victims, part, n_chunks, out,
                                                           victims, unres);
    g_launches++;
    return cudaGetLastError();
}

template <int W, int POLICY>
static cudaError_t launch_drain_t(const NodeTable& nt, const PodView& pv, const DrainArgs& da, uint32_t r,
                                  const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    constexpr uint32_t SMEM = tile_smem_bytes<W, POLICY != KS_SCORE_LEFTOVER>();
    k_drain_scan<W, POLICY><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, SMEM, st>>>(nt, pv, da, part, g.tiles_per_chunk);
    k_drain_commit<W, POLICY><<<(pv.P + 7) / 8, 256, 0, st>>>(nt, pv, da, part, g.n_chunks, r);
    g_launches += 2;
    return cudaGetLastError();
}

cudaError_t launch_drain_round(const NodeTable& nt, const PodView& pv, const DrainArgs& da, int policy, uint32_t r,
                               const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        return with_policy(policy, [&](auto pol) {
            return launch_drain_t<W, decltype(pol)::value>(nt, pv, da, r, part, g, st);
        });
    });
}

template <int W, int POLICY>
static cudaError_t launch_fit_drain_t(const NodeTable& nt, const PodView& pv, const DrainArgs& da, const FitDrainArgs& fa,
                                      uint32_t r, const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    constexpr uint32_t SMEM = tile_smem_bytes<W, POLICY != KS_SCORE_LEFTOVER>();
    k_fit_drain_scan<W, POLICY, false><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS, SMEM, st>>>(nt, pv, da, fa, part,
                                                                                                   g.tiles_per_chunk);
    k_fit_drain_commit<W, POLICY><<<(pv.P + 7) / 8, 256, 0, st>>>(nt, pv, da, fa, part, g.n_chunks, r);
    g_launches += 2;
    return cudaGetLastError();
}

cudaError_t launch_fit_drain_round(const NodeTable& nt, const PodView& pv, const DrainArgs& da, const FitDrainArgs& fa,
                                   int policy, uint32_t r, const PartialView& part, const DirectGrid& g, cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        return with_policy(policy, [&](auto pol) {
            return launch_fit_drain_t<W, decltype(pol)::value>(nt, pv, da, fa, r, part, g, st);
        });
    });
}

cudaError_t launch_fit_drain_refusals(const NodeTable& nt, const PodView& pv, const DrainArgs& da,
                                      const FitDrainArgs& fa, const DirectGrid& g, cudaStream_t st) {
    if (pv.P == 0) return cudaSuccess;
    return with_label_width(nt.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        k_fit_drain_scan<W, KS_SCORE_LEFTOVER, true><<<dim3(g.pod_ctas, g.n_chunks), DIRECT_THREADS,
                                                       tile_smem_bytes<W, false>(), st>>>(nt, pv, da, fa, PartialView{},
                                                                                          g.tiles_per_chunk);
        g_launches++;
        return cudaGetLastError();
    });
}

} // namespace ks
