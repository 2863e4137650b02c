// mask_store_probe.cu — store-pattern probe for the mask pass (k_mask_rows) on one device; driven by bench_mask_store.py.
//
// Every pattern writes the same buffer of `rows` mask rows of `pitch` bytes (the c3 shape: 1M x 6400 B) and nothing else
// outside the probe's own arrays, so the patterns differ only in HOW the bytes go out:
//   P0  k_fill256's shape: grid-stride 128-bit stores, consecutive lanes on consecutive 16 bytes (ks_measure_write_bandwidth)
//   P1  k_mask_rows' store shape: 960-thread CTAs, one per SM; a warp iteration = a group of 8 pods, lanes (pod slot ps, tile
//       t) = 4 rows x 8 lanes, two pods per thread; 256-byte (pod, column block) items claimed 4 groups at a time through
//       one cursor per column block, CTAs hop to the block with the most work left; lane t stores its 32 bytes at +0, +16
//   P2  P1, whole-line order: lane t stores at 16 t, then at 128 + 16 t (each instruction fills one 128-byte line per pod)
//   P3  P2 with 512-byte / 1 KB column blocks
//   P4  P2 + one atomicAdd per pod and column block into a 4 MB count array
//   P5  P2 + the 16-byte pod record loads of k_mask_rows (16 MB array, once per pod and column block, one group ahead)
//   P6  P5 with the records staged in shared memory: one thread per CTA claims chunks of CHUNK groups and brings their
//       records into a two-slot ring by bulk async copies (L2 evict-last, as K2's record loads) a chunk ahead; the warps
//       take the chunk's groups round robin
// Output: one JSON line, {"pattern": [GB/s of every repetition, in launch order]}.  Patterns are alternated.
#include <cuda_runtime.h>

#include "../kube-scheduler-rs-reference_b200/csrc/ks_internal.cuh"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                            \
        }                                                                                       \
    } while (0)

constexpr uint32_t CURSOR_STRIDE = 32; // one cursor per 128-byte line, as in k_mask_rows
constexpr uint32_t CLAIM = 4;
constexpr uint32_t HOP_MIN = 256;
constexpr int THREADS = 960;
constexpr uint32_t SMEM_PIN = 150 * 1024; // as much shared memory as k_mask_rows' blob: one CTA per SM

__global__ void __launch_bounds__(256) k_fill256(uint8_t* __restrict__ dst, uint64_t n32, uint32_t v) {
    const uint64_t n16 = 2 * n32;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (uint64_t)gridDim.x * blockDim.x)
        asm volatile("st.global.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst + i * 16), "r"(v) : "memory");
}

__device__ __forceinline__ void st_ef(uint8_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d), "l"(pol)
                 : "memory");
}

struct Probe {
    uint8_t* mask;
    uint32_t pitch;     // bytes per row
    uint32_t n_groups;  // groups of 8 rows
    uint32_t ncb;       // column blocks of BLOCK bytes (the last one may be cut by the pitch)
    uint32_t* cursor;   // [ncb * CURSOR_STRIDE]
    uint32_t* cnt;      // [rows] (P4)
    const uint4* rec;   // [rows] (P5, P6)
};

// HALF: P1's store order; else whole lines.  RED: count atomics.  REC: record loads.
template <int BLOCK, bool HALF, bool RED, bool REC>
__global__ void __launch_bounds__(1024, 1) k_probe(const __grid_constant__ Probe pr) {
    __shared__ unsigned long long s_key;
    const uint32_t tid = threadIdx.x, t = tid & 7, ps = (tid >> 3) & 3, lane = tid & 31;
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    const uint32_t n = pr.n_groups, ncb = pr.ncb, last = n - 1;
    uint32_t cb = (uint32_t)((uint64_t)blockIdx.x * ncb / gridDim.x);
    for (;;) {
        __syncthreads();
        uint32_t* cursor = pr.cursor + (size_t)cb * CURSOR_STRIDE;
        auto claim = [&]() -> uint32_t { return lane == 0 ? atomicAdd(cursor, CLAIM) : 0u; };
        uint32_t base = __shfl_sync(0xffffffffu, claim(), 0);
        uint32_t next_raw = claim();
        uint4 nA = make_uint4(0, 0, 0, 0), nB = nA;
        auto fetch = [&](uint32_t j, uint4& a, uint4& b) {
            if (REC) {
                const uint4* rp = pr.rec + (size_t)min(j, last) * 8u + 2u * ps;
                a = __ldg(rp);
                b = __ldg(rp + 1);
            }
        };
        fetch(base, nA, nB);
        const uint32_t col = cb * BLOCK;
        while (base < n) {
            const uint32_t end = min(base + CLAIM, n);
            uint32_t next = 0;
            for (uint32_t j = base; j < end; j++) {
                const uint4 rA = nA, rB = nB;
                uint32_t jn = j + 1;
                if (jn == end) {
                    next = __shfl_sync(0xffffffffu, next_raw, 0);
                    jn = next;
                }
                fetch(jn, nA, nB);
#pragma unroll
                for (int q = 0; q < 2; q++) {
                    const uint32_t pod = j * 8u + 2u * ps + q;
                    const uint4 r = q ? rB : rA;
                    const uint32_t v = pod ^ (REC ? r.x ^ r.y ^ r.z ^ r.w : 0u);
                    uint8_t* row = pr.mask + (size_t)pod * pr.pitch;
                    if (HALF) {
                        uint8_t* dst = row + col + 32u * t;
                        st_ef(dst, v, v, v, v, pol);
                        st_ef(dst + 16, v, v, v, v, pol);
                    } else {
#pragma unroll
                        for (int k = 0; k < BLOCK / 128; k++) {
                            const uint32_t off = col + 128u * k + 16u * t;
                            if (BLOCK == 256 || off < pr.pitch) st_ef(row + off, v, v, v, v, pol);
                        }
                    }
                    if (RED) {
                        uint32_t c = v & 0xFFu;
                        c += __shfl_xor_sync(0xffffffffu, c, 1);
                        c += __shfl_xor_sync(0xffffffffu, c, 2);
                        c += __shfl_xor_sync(0xffffffffu, c, 4);
                        if (t == 0 && c) atomicAdd(pr.cnt + pod, c);
                    }
                }
            }
            base = next;
            if (base < n) next_raw = claim();
        }
        if (ncb == 1) break;
        __syncthreads();
        if (tid == 0) s_key = 0;
        __syncthreads();
        for (uint32_t c = tid; c < ncb; c += blockDim.x) {
            const uint32_t used = *reinterpret_cast<volatile uint32_t*>(pr.cursor + (size_t)c * CURSOR_STRIDE);
            const uint32_t left = used < n ? n - used : 0u;
            if (left >= HOP_MIN || (left > 0 && used == 0)) {
                const uint32_t dist = (c + ncb - cb) % ncb;
                atomicMax(&s_key, ((unsigned long long)left << 32) | (0xFFFFFFFFu - dist));
            }
        }
        __syncthreads();
        const unsigned long long key = s_key;
        if (key == 0) break;
        cb = (cb + (0xFFFFFFFFu - (uint32_t)key)) % ncb;
    }
}

// P6: P5's stores and record dependence, with the records staged in a ring of RING slots of C groups (slot x % RING holds
// the CTA's x-th chunk; thread 0 claims and copies chunk x + 1 when warp 0 starts chunk x).
constexpr uint32_t RING = 2;
constexpr uint32_t CHUNK = 32; // 16-32 measured equally fast at the c3 shape, 64 slower (BASELINE.md)
__global__ void __launch_bounds__(1024, 1) k_probe_ring(const __grid_constant__ Probe pr, uint32_t C) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[RING], empty[RING];
    __shared__ uint32_t s_base[RING];
    __shared__ unsigned long long s_key;
    const uint32_t tid = threadIdx.x, t = tid & 7, ps = (tid >> 3) & 3, lane = tid & 31, warp = tid >> 5;
    const uint32_t nwarps = blockDim.x >> 5;
    uint64_t pol, pol_rec;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_rec));
    if (tid == 0) {
        for (uint32_t s = 0; s < RING; s++) {
            ks::mbar_init(&full[s], 1);
            ks::mbar_init(&empty[s], nwarps);
        }
        ks::fence_mbar_init();
    }
    const uint32_t n = pr.n_groups, ncb = pr.ncb;
    uint32_t cb = (uint32_t)((uint64_t)blockIdx.x * ncb / gridDim.x);
    uint32_t seq = 0, pending = 0; // chunks begun by this CTA; thread 0: the claim for the next chunk
    bool prod_done = false;
    for (;;) {
        __syncthreads();
        uint32_t* cursor = pr.cursor + (size_t)cb * CURSOR_STRIDE;
        auto issue = [&](uint32_t x) { // thread 0
            const uint32_t s = x % RING;
            ks::mbar_wait(&empty[s], ((x / RING) & 1u) ^ 1u);
            const uint32_t b = pending;
            s_base[s] = b;
            if (b < n) {
                const uint32_t bytes = min(C, n - b) * 128u;
                ks::fence_proxy_async();
                ks::mbar_arrive_expect_tx(&full[s], bytes);
                ks::tma_bulk_g2s(ring + (size_t)s * C * 128u, pr.rec + (size_t)b * 8u, bytes, &full[s], pol_rec);
                pending = atomicAdd(cursor, C);
            } else {
                ks::mbar_arrive(&full[s]);
                prod_done = true;
            }
        };
        if (tid == 0) {
            pending = atomicAdd(cursor, C);
            prod_done = false;
            issue(seq);
        }
        uint32_t j = seq, i = warp, base = 0, cnt = 0;
        auto enter = [&]() {
            if (tid == 0 && !prod_done) issue(j + 1);
            ks::mbar_wait(&full[j % RING], (j / RING) & 1u);
            base = s_base[j % RING];
            cnt = base < n ? min(C, n - base) : 0u;
        };
        auto settle = [&]() { // moves (j, i) to this warp's next group; false at the block's end chunk
            while (i >= cnt && cnt != 0) {
                __syncwarp();
                if (lane == 0) ks::mbar_arrive(&empty[j % RING]);
                i = i >= C ? i - C : 0u;
                j++;
                enter();
            }
            return cnt != 0;
        };
        auto rec = [&](uint32_t q) {
            return *reinterpret_cast<const uint4*>(ring + ((size_t)(j % RING) * C + i) * 128u + (2u * ps + q) * 16u);
        };
        enter();
        const uint32_t col = cb * 256u;
        bool more = settle();
        uint4 nA = more ? rec(0) : make_uint4(0, 0, 0, 0), nB = more ? rec(1) : nA;
        while (more) {
            const uint4 rA = nA, rB = nB;
            const uint32_t g = base + i;
            i += nwarps;
            more = settle();
            if (more) {
                nA = rec(0);
                nB = rec(1);
            }
#pragma unroll
            for (int q = 0; q < 2; q++) {
                const uint32_t pod = g * 8u + 2u * ps + q;
                const uint4 r = q ? rB : rA;
                const uint32_t v = pod ^ r.x ^ r.y ^ r.z ^ r.w;
                uint8_t* row = pr.mask + (size_t)pod * pr.pitch;
                st_ef(row + col + 16u * t, v, v, v, v, pol);
                st_ef(row + col + 128u + 16u * t, v, v, v, v, pol);
            }
        }
        __syncwarp();
        if (lane == 0) ks::mbar_arrive(&empty[j % RING]); // the end chunk
        seq = j + 1;
        if (ncb == 1) break;
        __syncthreads();
        if (tid == 0) s_key = 0;
        __syncthreads();
        for (uint32_t c = tid; c < ncb; c += blockDim.x) {
            const uint32_t used = *reinterpret_cast<volatile uint32_t*>(pr.cursor + (size_t)c * CURSOR_STRIDE);
            const uint32_t left = used < n ? n - used : 0u;
            if (left >= HOP_MIN || (left > 0 && used == 0)) {
                const uint32_t dist = (c + ncb - cb) % ncb;
                atomicMax(&s_key, ((unsigned long long)left << 32) | (0xFFFFFFFFu - dist));
            }
        }
        __syncthreads();
        const unsigned long long key = s_key;
        if (key == 0) break;
        cb = (cb + (0xFFFFFFFFu - (uint32_t)key)) % ncb;
    }
}

static void launch_ring(Probe pr, int sms, cudaStream_t st) {
    CK(cudaFuncSetAttribute(k_probe_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_PIN));
    pr.ncb = (pr.pitch + 255) / 256;
    CK(cudaMemsetAsync(pr.cursor, 0, (size_t)pr.ncb * CURSOR_STRIDE * 4, st));
    k_probe_ring<<<sms, THREADS, SMEM_PIN, st>>>(pr, CHUNK);
    CK(cudaGetLastError());
}

template <int BLOCK, bool HALF, bool RED, bool REC>
static void launch(Probe pr, int sms, cudaStream_t st) {
    auto k = k_probe<BLOCK, HALF, RED, REC>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_PIN));
    pr.ncb = (pr.pitch + BLOCK - 1) / BLOCK;
    CK(cudaMemsetAsync(pr.cursor, 0, (size_t)pr.ncb * CURSOR_STRIDE * 4, st));
    k<<<sms, THREADS, SMEM_PIN, st>>>(pr);
    CK(cudaGetLastError());
}

int main(int argc, char** argv) {
    const uint32_t rows = argc > 1 ? (uint32_t)atoi(argv[1]) : 1000000u;
    const uint32_t pitch = argc > 2 ? (uint32_t)atoi(argv[2]) : 6400u;
    const int reps = argc > 3 ? atoi(argv[3]) : 7;
    if (rows % 8 || pitch % 256) {
        fprintf(stderr, "rows must be a multiple of 8 and pitch of 256\n");
        return 1;
    }
    int dev = 0, sms = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t bytes = (size_t)rows * pitch;
    Probe pr{};
    pr.pitch = pitch;
    pr.n_groups = rows / 8;
    CK(cudaMalloc(&pr.mask, bytes));
    const size_t cursor_bytes = ((size_t)pitch / 256 + 1) * CURSOR_STRIDE * 4; // one cursor per column block of >= 256 B
    CK(cudaMalloc(&pr.cursor, cursor_bytes));
    CK(cudaMalloc(&pr.cnt, (size_t)rows * 4));
    uint4* rec = nullptr;
    CK(cudaMalloc(&rec, (size_t)rows * 16));
    CK(cudaMemset(rec, 0x5A, (size_t)rows * 16));
    CK(cudaMemset(pr.cnt, 0, (size_t)rows * 4));
    pr.rec = rec;
    cudaStream_t st;
    CK(cudaStreamCreate(&st));
    struct Pat {
        const char* name;
        void (*run)(Probe, int, cudaStream_t);
    };
    const Pat pats[] = {
        {"P0_fill", [](Probe p, int s, cudaStream_t q) { k_fill256<<<s * 8, 256, 0, q>>>(p.mask, (uint64_t)p.pitch * p.n_groups * 8 / 32, 0x3C3C3C3Cu); }},
        {"P1_k2_half_lines", [](Probe p, int s, cudaStream_t q) { launch<256, true, false, false>(p, s, q); }},
        {"P2_whole_lines", [](Probe p, int s, cudaStream_t q) { launch<256, false, false, false>(p, s, q); }},
        {"P3_whole_lines_512B", [](Probe p, int s, cudaStream_t q) { launch<512, false, false, false>(p, s, q); }},
        {"P3_whole_lines_1KB", [](Probe p, int s, cudaStream_t q) { launch<1024, false, false, false>(p, s, q); }},
        {"P4_whole_lines_red", [](Probe p, int s, cudaStream_t q) { launch<256, false, true, false>(p, s, q); }},
        {"P5_whole_lines_rec", [](Probe p, int s, cudaStream_t q) { launch<256, false, false, true>(p, s, q); }},
        {"P6_whole_lines_rec_ring", launch_ring},
    };
    const int np = (int)(sizeof(pats) / sizeof(pats[0]));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int p = 0; p < np; p++) pats[p].run(pr, sms, st); // warm-up: module load, first touch of every page
    CK(cudaStreamSynchronize(st));
    std::vector<std::vector<double>> gbs(np);
    for (int r = 0; r < reps; r++)
        for (int p = 0; p < np; p++) {
            CK(cudaMemsetAsync(pr.cursor, 0, cursor_bytes, st));
            CK(cudaEventRecord(e0, st));
            pats[p].run(pr, sms, st);
            CK(cudaEventRecord(e1, st));
            CK(cudaEventSynchronize(e1));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            gbs[p].push_back(bytes / (ms * 1e-3) / 1e9);
        }
    // spot check of the last pattern only (P6, which follows P0 fill): on 3 rows, the first 4 bytes of every 16 no longer
    // hold the fill value
    std::vector<uint8_t> h(pitch);
    for (uint32_t row : {0u, rows / 2 + 3, rows - 1}) {
        CK(cudaMemcpy(h.data(), pr.mask + (size_t)row * pitch, pitch, cudaMemcpyDeviceToHost));
        for (uint32_t i = 0; i < pitch; i += 16)
            if (h[i] == 0x3C && h[i + 1] == 0x3C && h[i + 2] == 0x3C && h[i + 3] == 0x3C) { // P6 writes the row index
                fprintf(stderr, "row %u byte %u not written by the last pattern\n", row, i);
                return 1;
            }
    }
    printf("{\"sms\": %d, \"rows\": %u, \"pitch\": %u, \"bytes\": %zu, \"gbs\": {", sms, rows, pitch, bytes);
    for (int p = 0; p < np; p++) {
        printf("%s\"%s\": [", p ? ", " : "", pats[p].name);
        for (size_t r = 0; r < gbs[p].size(); r++) printf("%s%.1f", r ? ", " : "", gbs[p][r]);
        printf("]");
    }
    printf("}}\n");
    CK(cudaFree(pr.mask));
    CK(cudaFree(pr.cursor));
    CK(cudaFree(pr.cnt));
    CK(cudaFree(rec));
    return 0;
}
