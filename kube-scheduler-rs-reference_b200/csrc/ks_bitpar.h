// ks_bitpar.h — bit-parallel fast path (ks_bitpar.cu).
//
// Idea: `req <= free` depends only on ORDER.  Nodes are ranked once per snapshot (global position of each
// node in ascending free_cpu / free_mem order); a pod's request becomes a global rank threshold (binary
// search once per pod).  For a tile of 256 nodes the feasible bits of one resource are then a row of a
// prefix table indexed by the tile-local rank of the threshold, and the tile-local rank is
//   base[bucket][tile] + popc(member[bucket][tile] & lowmask)
// (bucket = 64 consecutive global positions).  Label selectors are ANDs of per-(key,value) node columns.
// Three tile indexes are built per snapshot, all in the column-block format below: node order for the mask kernel
// (k_mask_rows), descending priority order for the LEFTOVER argmax and descending score-bound order for the
// LeastAllocated argmax.  The mask kernel takes tile-local ranks from rank tables that hold the rank of every possible
// threshold ([column block][threshold][tile pair] u32, read through L1/L2); one pod takes 8 lanes = 256 contiguous bytes
// of its mask row, lane t granules t and 8 + t (each store instruction writes one whole 128-byte line per pod): ~50
// instructions per 256 cells.  The argmax kernels derive the rank with the base + popc formula from the bucket arrays of
// their order.  KS_SCORE_LEFTOVER is separable (node part - pod part), so argmax-score is the first feasible node in a
// static priority order: a short early-exit scan per pod (k_first_fit).
#pragma once
#include "ks_internal.cuh"

namespace ks {

constexpr int BP_TILE = 256;          // nodes per tile = 8 mask words = one 32-byte row
constexpr int BP_ROWS = BP_TILE + 1;  // prefix-table rows per tile and resource (local rank 0..256)
constexpr int BP_THREADS = 1024;
constexpr int BP_SMEM_MAX = 232448;   // 227 KB opt-in limit per CTA

// Column-block format: column block = 8 tiles (2048 slots of the index's order); tile k is position k % 8 of column
// block k / 8.  One blob per column block:
//   tabC [257 rows][256 B], tabM [257 rows][256 B], pairs [64*W bits][256 B]
// and every 256-byte line is [tile 0 | tile 1 | ... | tile 7] (32 B each) = 16 granules of 16 B.  Lane t of an 8-lane
// shared-memory phase reads granule t (tile t/2) of the row of its tile's rank, then granule 8 + t (tile 4 + t/2) of
// another row: offsets 16 t modulo 128 -> 8 distinct bank groups for any ranks.  Tiles past the last node are built too,
// with all-zero rows and columns.
constexpr uint32_t RW_TILES = 8;                            // tiles per column block
constexpr uint32_t RW_LINE = 256;                           // bytes per table row / pair column of a column block
constexpr uint32_t RW_TAB_BYTES = (uint32_t)BP_ROWS * RW_LINE; // 65792

struct RowsLayout { // of all three indexes (make_layout_rows)
    uint32_t ncb;        // column blocks
    uint32_t n_tiles;    // ceil(N / 256)
    uint32_t off_tabC, off_tabM, off_pairs; // byte offsets inside a column-block blob
    uint32_t smem_bytes; // bytes staged in shared memory (tables, + pair columns when they fit)
    uint32_t cb_stride;  // bytes between two column-block blobs in global memory
    uint32_t pairs_smem; // 1 = the pair columns are staged with the tables, 0 = read through L1/L2 (W = 8)
    uint32_t n_thr;      // thresholds per column block in the rank tables: N + 1
};

// The bucket arrays of one ordered index, [resource][bucket][tile] (resource 0 = cpu, 1 = memory), with (N >> 6) + 1
// buckets of 64 global positions and n_tiles tiles (none for the padding tiles).  The tile-local rank of threshold g in
// tile k is
//   base[r][g >> 6][k] + popc(memb[r][g >> 6][k] & ((1 << (g & 63)) - 1)).
struct TileBuckets {
    uint16_t* base[2];
    unsigned long long* memb[2];
};

// The node order of a bound-ordered argmax (k_least_alloc, k_most_alloc, k_least_balanced): every node's score bound,
// the tile index and evaluation rows in descending bound order.  LEAST_ALLOCATED's is built by bitpar_build, the others
// on the first call that needs them after each bitpar_build (bitpar_prepare_order).
struct BoundOrder {
    DevBuf b;       // [int64 Nord] bound of every node in descending order (ties by index); padding: INT64_MIN for
                    // LEAST_ALLOCATED, -1 for the others
    DevBuf idx;     // [int32 Nord]
    DevBuf eval;    // [NodeEval Nord] per slot of that order: what the exact score needs
    DevBuf blob;    // lay_r.ncb column-block blobs in that order, read through L1/L2 by the walk
    DevBuf buckets; // TileBuckets of blob
    DevBuf sort;    // [uint32 2N] sort scratch, then [int64 2] smallest positive allocatable cpu / memory (8-aligned);
                    // not allocated for LEAST_ALLOCATED, whose order k_node_rank writes
    bool valid = false; // matches the current index
};

// The index of one snapshot.  Device arrays (element type in brackets) are grow-only buffers, read through .as<T>().
// Owned by the snapshot and freed with it, with the snapshot's device current.
struct BitparIndex {
    DevBuf sortedC;   // [int64 N] free_cpu ascending
    DevBuf sortedM;   // [int64 N] free_mem ascending
    DevBuf gposC;     // [uint32 N] position of node n in sortedC (ties by node index)
    DevBuf gposM;
    DevBuf ord_prio;  // [int64 Nord] nodes in descending priority order (ties by node index), padded to a tile
    DevBuf ord_idx;   // [int32 Nord]
    DevBuf splC;      // [int64] every `spl_stride`-th element of sortedC / sortedM (<= RANK_SPLITTERS = 8192 splitters)
    DevBuf splM;
    DevBuf blobP;     // lay_r.ncb column-block blobs in priority order (tile k = priority ranks 256k..), read through
                      // L1/L2 by k_first_fit_head / _tail
    DevBuf bucketsP;  // TileBuckets of blobP (tile_buckets)
    DevBuf pod_ranks; // [uint2 P] per-call scratch
    DevBuf tail_list; // [uint32 P + 1] per-call scratch: pods left for k_first_fit_tail, then the count at word P
    BoundOrder ordL;  // KS_SCORE_LEAST_ALLOCATED (k_least_alloc)
    DevBuf hintL;     // [float4 Nord] per slot of ordL: single-precision score model (pre-filter of k_least_alloc)
    BoundOrder ordM;  // KS_SCORE_MOST_ALLOCATED (k_most_alloc), built lazily
    BoundOrder ordB;  // KS_SCORE_LEAST_BALANCED (k_least_balanced), built lazily
    DevBuf live;      // [uint64 KS_MAX_LABEL_WORDS + 2] label bits carried by at least one node, max allocatable cpu, memory
    DevBuf rec_s;     // [uint4] rows kernel: {threshold_cpu, threshold_mem, pod index, selector columns} per pod, P rounded up to 8
    DevBuf blobR;     // rows kernel: lay_r.ncb column-block blobs in node order
    DevBuf rank;      // [uint32] rows kernel: [cb][threshold g][resource][j] = nodes of tile j (low 16 bits) and tile j + 4
                      // (high 16 bits) at sorted positions < g
    DevBuf tile_sorted; // [uint32] build scratch: per tile, its nodes' global positions in ascending order
    RowsLayout lay_r{}; // the layout of blobR, blobP and every BoundOrder's blob
    DevBuf rk_hist;   // [uint32] node sample sort scratch: per order 256 bucket counts, splitters, per-node bucket / slot, lists
    DevBuf rk_spl_v;
    DevBuf rk_spl_i;
    DevBuf rk_bkt;
    DevBuf rk_loc;
    DevBuf rk_perm;
    uint32_t N = 0, Nord = 0, W = 0, spl_stride = 1, n_spl = 0;
    bool valid = false;
    int sms = 0;
    Stream aux; // the argmax kernels run here, overlapped with k_mask_rows
    Event ev_fork, ev_join;
    DevBuf cursor; // [uint32 ncb * RW_CURSOR_STRIDE] work cursors of the mask kernel (k_mask_rows), zeroed by k_pod_ranks
    DevBuf trace;  // KS_TRACE=1: per-kernel %globaltimer stamps of the last select (ks_last_trace)
    ~BitparIndex(); // detaches the kernels from a trace buffer this index owns
};
constexpr int BP_TRACE_WORDS = 16;

cudaError_t bitpar_build(BitparIndex& ix, const NodeTable& nt, int64_t* prio, cudaStream_t st);
bool bitpar_profitable(const BitparIndex& ix, uint32_t P);
cudaError_t bitpar_prepare(BitparIndex& ix, uint32_t P);
// The order of `policy' (KS_SCORE_MOST_ALLOCATED, KS_SCORE_LEAST_BALANCED; a no-op for the others): built on the first
// call after each bitpar_build that needs it (enqueued on st; must run before a stream-captured bitpar_select), a no-op
// after that
cudaError_t bitpar_prepare_order(BitparIndex& ix, const NodeTable& nt, int policy, cudaStream_t st);
cudaError_t bitpar_select(BitparIndex& ix, SelectLaunch& L, cudaEvent_t before_mask, cudaEvent_t after_mask);
// slots of ks_last_trace (include/ksched.h); cudaErrorNotSupported unless the index was created under KS_TRACE=1
cudaError_t bitpar_read_trace(const BitparIndex& ix, unsigned long long out_ns[BP_TRACE_WORDS]);

} // namespace ks
