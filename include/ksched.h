/* ksched.h — C ABI of the H100 scheduling core (libksched.so).
 *
 * Drop-in boundary for the hot path of acrlabs/kube-scheduler-rs-reference.  The reference is a binary
 * crate with no FFI; the three in-crate functions this library replaces are (paths relative to
 * /root/reference):
 *   check_node_validity(&Pod,&Node,&Context) -> Result<(),InvalidNodeReason>   src/predicates.rs:63-77
 *   select_node_for_pod(&Pod,&Context) -> Option<Node>                         src/main.rs:51-71
 *   Context{client,node_store} (node cache + per-cell LIST of bound pods)      src/util.rs:12-15,
 *                                                                              src/predicates.rs:21-38
 * A Rust host would bind these entry points with an `extern "C"` block (INTEGRATION.md shows it);
 * signatures use only plain pointers, sizes and opaque handles.  No torch / C++ types cross the ABI.
 *
 * Units: cpu = int64 millicores, memory = int64 bytes, labels = W x uint64 bit columns per row
 * (bit set on a node = node carries that (key,value) pair; bit set on a pod = selector requires it).
 * Cell semantics (bit-exact with oracle/oracle.c):
 *   fit   = req_cpu <= free_cpu && req_mem <= free_mem          (src/predicates.rs:42, non-strict)
 *   match = for all w: (sel[w] & ~labels[w]) == 0               (src/predicates.rs:45-61)
 *   code  = !fit ? 1 : !match ? 2 : 0                           (src/predicates.rs:68-76, fit first)
 * All functions return KS_OK (0) or a negative KS_ERR_*; nothing aborts or throws across the ABI
 * (the reference panics on malformed data, src/predicates.rs:29,31,36).  ks_last_error() returns a
 * thread-local description of the most recent failure on the calling thread.
 */
#ifndef KSCHED_H
#define KSCHED_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KS_OK 0
#define KS_ERR_INVALID (-1)
#define KS_ERR_CUDA (-2)
#define KS_ERR_PARSE (-3)
#define KS_ERR_NOMEM (-4)
#define KS_ERR_RANGE (-5)
#define KS_ERR_INEXACT (-6)
#define KS_ERR_MISSING (-7)
#define KS_ERR_NO_DEVICE (-8)

/* cell codes = Ok(()) / InvalidNodeReason (src/predicates.rs:14-18) */
#define KS_CELL_OK 0
#define KS_CELL_NOT_ENOUGH_RESOURCES 1
#define KS_CELL_NODE_SELECTOR_MISMATCH 2

/* score policies (spec extension — the reference has no score; DESIGN.md "Score") */
#define KS_SCORE_LEFTOVER 0        /* (free_cpu-req_cpu)*2^22 + (free_mem-req_mem); separable => static node order */
#define KS_SCORE_LEAST_ALLOCATED 1 /* ((free_cpu-req_cpu)*100/alloc_cpu + (free_mem-req_mem)*100/alloc_mem)/2, floor */
/* 2 is reserved and rejected as a policy. */
/* KS_SCORE_MOST_ALLOCATED: bin-packing, upstream NodeResourcesFit's MostAllocated strategy with weights 1 and 1.  Per
 * resource, with allocatable A, free f and request q:
 *   term(f, A, q) = A > 0 ? clamp(A - (f - q), 0, A) * 100 / A : 0     (int64, truncating division of a value >= 0)
 *   score         = (term(free_cpu, alloc_cpu, req_cpu) + term(free_mem, alloc_mem, req_mem)) / 2,   in [0, 100]
 * A - (f - q) is upstream's `requested` (the bound pods' requests plus this pod's); upstream clamps it to A, and the
 * lower clamp covers free > allocatable, which negative bound requests or releases can leave here.  Like
 * KS_SCORE_LEAST_ALLOCATED, pods without requests are scored as requesting 0: upstream's non-zero defaults (100m CPU,
 * 200 MB memory) are not added.  Every call that takes a policy takes this one, and ks_select runs it on both kernel
 * paths; its bit-parallel order is built on the first call that needs it after each snapshot change. */
#define KS_SCORE_MOST_ALLOCATED 3
/* KS_SCORE_LEAST_BALANCED: upstream's default resource scoring, NodeResourcesFit (LeastAllocated) plus
 * NodeResourcesBalancedAllocation, each with weight 1, for cpu and memory.  With allocatable A, free f and request q:
 *   least    = the KS_SCORE_LEAST_ALLOCATED score, in [0, 100] on feasible cells
 *   u_r      = clamp(A_r - (f_r - q_r), 0, A_r)                            (int64, as KS_SCORE_MOST_ALLOCATED)
 *   x_r      = (double)u_r / (double)A_r for each resource with A_r > 0 (each operand rounded to nearest even, then
 *              one IEEE division; a resource with A_r <= 0 is skipped)
 *   std      = |x_cpu - x_mem| / 2 when both resources are kept, else 0
 *   balanced = (int64) trunc((1 - std) * 100), each operation one IEEE double operation rounded to nearest, in [0, 100]
 *   score    = least + balanced,   in [0, 200]
 * Every kernel path computes `balanced' with the same correctly rounded operations (no FMA contraction, no reciprocal),
 * so every call returns the same score bit for bit.  Departures from upstream: its non-zero request defaults are not
 * added, u has a lower clamp (free > allocatable), and ties go to the lowest node index instead of a random one.  Every
 * call that takes a policy takes this one.  ks_select runs it on both kernel paths, and KS_SELECT_AUTO chooses between
 * them by the same P * N >= 2^24 rule as for the other policies; its bit-parallel order is built on the first call that
 * needs it after each snapshot change.  ks_place_replicas places its copies one at a time (see there). */
#define KS_SCORE_LEAST_BALANCED 4

/* where caller-owned buffers live */
#define KS_MEM_HOST 0
#define KS_MEM_DEVICE 1

/* ks_select flags */
#define KS_SELECT_AUTO 0u
#define KS_SELECT_FORCE_DIRECT 1u  /* per-cell kernel (any policy) */
#define KS_SELECT_FORCE_BITPAR 2u  /* bit-parallel kernel (any policy) */
#define KS_SELECT_TIMING 4u        /* record CUDA events around each kernel; read with ks_last_timings */
#define KS_SELECT_NO_GRAPH 8u      /* all-device calls are replayed from a cached CUDA graph; this disables it */

/* value limits that keep scores and sums inside int64.  Every node's free value stays within +-KS_MAX_CPU_MILLI /
 * +-KS_MAX_MEM_BYTES: allocatable and bound pods are checked by set_nodes / set_bound, a bind by apply_bind (against
 * the node's free after it), and every call that commits requests against free[] (ks_snapshot_commit_claims,
 * ks_stream_bind, ks_gang_bind, ks_stream_submit) takes requests in [0, limit] only, so an accepted request leaves its
 * node's free in [0, free]; anything else is KS_ERR_RANGE before any change.  Pending pods of the calls that change
 * nothing (ks_select, ks_explain, ks_select_topk, ks_preempt, ks_check_cell(s), ks_select_sampling) are NOT checked:
 * device-space pods could not be without an extra pass.  Outside +-limit their scores are undefined. */
#define KS_MAX_CPU_MILLI ((int64_t)1 << 36)
#define KS_MAX_MEM_BYTES ((int64_t)1 << 55)
#define KS_MAX_LABEL_WORDS 8u

typedef struct ks_snapshot ks_snapshot; /* replaces Context.node_store + the LIST, src/util.rs:12-15 */

typedef struct ks_pods { /* SoA view of P pending pods (what total_pod_resources + node_selector pack to) */
    uint64_t n;
    const int64_t* req_cpu;  /* [n] millicores   (src/util.rs:54-75 per pod) */
    const int64_t* req_mem;  /* [n] bytes */
    const uint64_t* sel;     /* [n*W] required label bits (all zero = no selector) */
    int32_t mem_space;       /* KS_MEM_HOST or KS_MEM_DEVICE for the three arrays above */
} ks_pods;

/* ---- multi-GPU exchange of the bindings (SURVEY.md section 8e; one process per GPU, pods sharded) ----
 * The reference has no multi-process story; north_star asks for ONE all-gather of the per-pod bindings.  Here the
 * all-gather is fused into the argmax kernels: every binding is stored into the local output AND into every peer's
 * gather buffer through peer-mapped (CUDA IPC) pointers over NVLink, then one flag per (source, destination) pair is
 * released; ks_select ends with a wait on this rank's flags, so when the call's stream work is done the gather
 * buffer holds the bindings of every rank.  No collective library call is on the data path.
 * All pointers are DEVICE pointers valid in the calling process (peer_* ones were opened with ks_ipc_open). */
#define KS_MAX_PEERS 15u
typedef struct ks_exchange {
    uint32_t world, rank;                 /* ranks taking part, this rank */
    uint32_t n_peers;                     /* = world - 1 */
    int32_t* peer_node_idx[KS_MAX_PEERS]; /* where THIS rank's node_idx[0..n) goes in peer k's gather buffer */
    int64_t* peer_score[KS_MAX_PEERS];    /* same for score */
    uint32_t* peer_flag[KS_MAX_PEERS];    /* peer k's arrival flag for THIS rank */
    uint32_t* local_flags;                /* this rank's flags [world]; entry r is written by rank r */
    uint32_t* local_state;                /* this rank's private words [16], zeroed, 8-byte aligned: [0] step sequence
                                             number, [1] CTA counter, [2..11] five 64-bit %globaltimer stamps (ns) of
                                             the last step: first argmax CTA, flags published, wait started, wait done,
                                             second argmax kernel started */
} ks_exchange;

typedef struct ks_bindings { /* outputs; any pointer may be NULL to skip that output */
    int32_t* node_idx;       /* [n] argmax-score feasible node, ties -> lowest index, -1 = NoNodeFound */
    int64_t* score;          /* [n] score of node_idx (0 when -1) */
    uint32_t* feasible_cnt;  /* [n] number of feasible nodes */
    int32_t mem_space;       /* space of the three arrays above */
    uint8_t* mask;           /* [n rows] feasible bit-mask, bit (n%8) of byte n/8 of the row */
    uint64_t mask_row_bytes; /* row pitch; multiple of 32, >= ks_mask_row_bytes(N); ks_mask_row_bytes_aligned(N) is fastest */
    int32_t mask_space;      /* space of mask (may differ: keep a 6 GB mask in HBM, bindings on host) */
    void* bindings_ready_event; /* optional cudaEvent_t (NULL = none), device-space outputs only: recorded as soon as
                                   node_idx and score are final - on the bit-parallel path that is well before the
                                   mask/count pass ends, so a collective over the bindings can overlap it */
    const ks_exchange* exchange; /* optional (NULL = none), device-space outputs only: fused all-gather, see above */
} ks_bindings;

const char* ks_last_error(void);
int ks_version(void);
int ks_device_count(void);           /* number of CUDA devices visible; 0 when none */
uint64_t ks_launch_count(void);      /* kernels launched by this library since load */
uint64_t ks_mask_row_bytes(uint32_t n_nodes); /* 32 * ceil(n_nodes/256): the smallest legal row pitch */
/* 256 * ceil(n_nodes/2048): the recommended pitch for a device-space mask.  The mask kernel writes one 256-byte block
 * per (pod, 2048-node column block); with this pitch (and a 256-byte-aligned base) every block is whole and aligned,
 * so no store straddles two 256-byte blocks of memory (on an H100 at 1M pods x 50k nodes the minimal pitch made that
 * kernel 8 % slower when each store instruction wrote half lines, 4 % slower with whole-line stores).  Bytes of a row
 * beyond ks_mask_row_bytes(n_nodes) carry no information: up to the aligned size the bit-parallel path writes them
 * as zeros (whole 32-byte tiles that fit the pitch), the per-cell path leaves them untouched. */
uint64_t ks_mask_row_bytes_aligned(uint32_t n_nodes);

/* ---- snapshot: device-resident node table (replaces node_store.state(), src/main.rs:56) ---- */
int ks_snapshot_create(int device, ks_snapshot** out);
void ks_snapshot_destroy(ks_snapshot* s);
/* host arrays; labels = [n_nodes*label_words]; resets bound load (free = alloc). */
int ks_snapshot_set_nodes(ks_snapshot* s, uint32_t n_nodes, uint32_t label_words, const int64_t* alloc_cpu,
                          const int64_t* alloc_mem, const uint64_t* labels);
/* K0: free[n] = alloc[n] - sum over bound pods on n (src/predicates.rs:27-38).  host arrays. */
int ks_snapshot_set_bound(ks_snapshot* s, uint64_t n_bound, const int32_t* node_idx, const int64_t* req_cpu,
                          const int64_t* req_mem);
/* incremental: one more pod bound to node_idx (what the next LIST would show after src/main.rs:103).  A negated
 * request releases it.  KS_ERR_RANGE, and free[] unchanged, for a request outside +-limit or a bind that would leave
 * the node's free outside +-limit. */
int ks_snapshot_apply_bind(ks_snapshot* s, int32_t node_idx, int64_t req_cpu, int64_t req_mem);
int ks_snapshot_get_free(ks_snapshot* s, int64_t* free_cpu, int64_t* free_mem); /* D2H, [n_nodes] each */
uint32_t ks_snapshot_num_nodes(const ks_snapshot* s);
uint32_t ks_snapshot_label_words(const ks_snapshot* s);

/* ---- device memory that other processes of the node can map (CUDA IPC), for ks_exchange ----
 * ks_ipc_alloc: cudaMalloc + zero fill on `device`; out_handle receives the 64-byte cudaIpcMemHandle_t to send to the
 * peers (any byte transport: torch.distributed, MPI, a file).  ks_ipc_open maps a peer's allocation into this process
 * (peer access between the two GPUs is enabled by the runtime).  ks_ipc_close / ks_ipc_free undo them. */
/* after a run of ks_select calls with an exchange: synchronises the device and reports whether any wait timed out */
int ks_exchange_check(ks_snapshot* s);
int ks_ipc_alloc(int device, uint64_t bytes, void** out_ptr, uint8_t out_handle[64]);
int ks_ipc_open(int device, const uint8_t handle[64], void** out_ptr);
int ks_ipc_close(int device, void* ptr);
int ks_ipc_free(int device, void* ptr);
/* store-only bandwidth of the device: best of `iters` passes of a plain coalesced 128-bit-store fill over dev_buf
 * (bytes >= 1 MiB, 32-byte aligned; its contents are overwritten).  MEASURED_PEAKS-style HBM peaks are copies
 * (read + write bytes); a kernel that only writes - the feasible-mask pass - is bounded by this figure instead. */
int ks_measure_write_bandwidth(int device, void* dev_buf, uint64_t bytes, int iters, double* out_gbs);
/* synchronising device-to-host copy of `bytes` bytes (reading a gather buffer allocated with ks_ipc_alloc) */
int ks_device_read(int device, const void* dev_ptr, void* host_ptr, uint64_t bytes);

/* ---- per-cell entry = check_node_validity (src/predicates.rs:63-77) ---- */
int ks_check_cell(ks_snapshot* s, int64_t req_cpu, int64_t req_mem, const uint64_t* sel, uint32_t node_idx);
/* K1: all P*N reason codes, out_codes[p*N+n] in host memory (small problems / parity tests) */
int ks_check_cells(ks_snapshot* s, const ks_pods* pods, uint8_t* out_codes);

/* ---- per-pod batched entry = select_node_for_pod over P pods ("predicates::run") ---- */
int ks_select(ks_snapshot* s, const ks_pods* pods, int policy, uint32_t flags, ks_bindings* out,
              void* cuda_stream /* cudaStream_t or NULL = library stream; call returns after completion
                                   for host-space outputs, after enqueue for all-device outputs */);
/* milliseconds of the kernels of the last KS_SELECT_TIMING call on this snapshot:
 * ms[0]=dominant mask/score kernel, ms[1]=argmax scan / combine, ms[2]=total enqueue-to-done. */
int ks_last_timings(ks_snapshot* s, float ms[3]);
/* name of the dominant kernel path the last ks_select used: "direct" or "bitpar" */
const char* ks_last_path(const ks_snapshot* s);
/* Timeline of the last bit-parallel ks_select on this snapshot, from %globaltimer stamps written by the kernels
 * themselves (the streams of a step overlap, which per-kernel profilers serialise).  Only when the process runs with
 * KS_TRACE=1 in its environment (else KS_ERR_INVALID); synchronises the device.  out_ns[k], nanoseconds of the
 * device clock, 0 = kernel did not run:  0/1 pod-rank kernel first CTA start / last CTA end, 2/3 first argmax kernel,
 * 4/5 second argmax kernel, 6/7 mask kernel, 8 end of the mask CTA that finished first; 9..15 reserved (0). */
int ks_last_trace(ks_snapshot* s, uint64_t out_ns[16]);

/* ---- streaming reconcile (BASELINE.json config C5): micro-batches against the resident snapshot ----
 * The reference re-LISTs bound pods for every cell (src/predicates.rs:34), so a pod always sees earlier binds.
 * A batched pass sees one snapshot, so two pods of a batch may claim the same capacity.  K3 resolves that:
 * claims are taken per node in arrival (array) order; a claim is accepted iff its request still fits what is
 * left on the node, and then decrements it.  Capacity never goes negative through this path.
 *
 * ks_snapshot_commit_claims: host arrays; claim i = pod i wants node claim_node[i] (-1 = no claim).
 *   out_accepted[i] = 1/0.  Accepted requests are subtracted from free[] on the device (same effect as
 *   ks_snapshot_apply_bind per accepted claim).  Every replica that commits the same claim list in the same
 *   order ends with the same free[] (multi-GPU streaming: all-gather the claims, commit everywhere).
 * ks_stream_bind: the full micro-batch loop on one GPU — select (per-cell kernel, any policy) for the pending
 *   pods, commit, re-select the losers against the updated free[], until every pod is bound or has no feasible
 *   node.  out_node_idx[i] = bound node or -1 (= ReconcileError::NoNodeFound, src/main.rs:116-118).
 * Both take requests in [0, KS_MAX_CPU_MILLI] / [0, KS_MAX_MEM_BYTES] only (every claim, every pod; -1 claims too):
 * KS_ERR_RANGE before any device work otherwise. */
int ks_snapshot_commit_claims(ks_snapshot* s, uint64_t n_claims, const int32_t* claim_node, const int64_t* req_cpu,
                              const int64_t* req_mem, uint8_t* out_accepted);
int ks_stream_bind(ks_snapshot* s, const ks_pods* pods /* host space */, int policy, int32_t* out_node_idx,
                   int64_t* out_score, uint32_t* out_rounds);

/* ---- pod groups, all-or-nothing (gang scheduling; upstream's coscheduling PodGroup minMember; spec extension,
 * DESIGN.md 5e) ----
 * Pods arrive in array order and are cut into groups: group g is the pods [offset[g], offset[g+1]), 1 to
 * KS_GANG_MAX_SIZE of them, with 0 <= min_member[g] <= its size.  Groups run in order, each against free[] as the
 * earlier groups left it:
 *   1. the ks_stream_bind micro-batch loop runs over the group's pods, unchanged: every round selects against the
 *      current free[] under `policy`, claims are accepted per node in arrival order while they fit, losers retry; the
 *      loop ends when no pod is pending (or after size + 2 rounds, which never binds);  placed[g] = pods it bound;
 *   2. placed[g] >= min_member[g]: the group commits; its placed pods keep their nodes and scores and stay charged,
 *      the others get -1 / 0 (NoNodeFound);
 *   3. otherwise it rolls back: every pod of the group gets -1 / 0 and free[] is restored bit for bit to its value
 *      before the group, so the next group sees exactly what this one saw.
 * So one group with min_member 0 is ks_stream_bind (same bindings, scores and final free[]), and singleton groups
 * give every pod the binds of all earlier pods (the reference's sequential reconcile, with the argmax).  Placement
 * inside a group is the stream loop's greedy, not a bin-packing search: a group can fail where another assignment
 * would have fitted (upstream coscheduling does not search either).
 * One H2D copy, one cooperative launch that walks every group on the device, one D2H copy.  Host-space pods and
 * outputs: out_node_idx[pods->n] (required when pods->n > 0), out_score[pods->n], out_placed[n] (before any
 * rollback) and out_rounds[n] may be NULL.  Checked before any device work: KS_ERR_INVALID for a NULL gangs or group
 * array, offset[0] != 0, decreasing offsets, offset[n] != pods->n, a bad policy or device-space pods;
 * KS_ERR_RANGE for a group of 0 or more than KS_GANG_MAX_SIZE pods, min_member above its size or a request outside
 * [0, limit] (as ks_stream_bind).  free[] changes, as
 * with ks_stream_bind.  An empty snapshot places nothing: every group with min_member >= 1 rolls back. */
#define KS_GANG_MAX_SIZE 1024u
typedef struct ks_gangs { /* host memory */
    uint64_t n;                  /* groups */
    const uint64_t* offset;      /* [n+1] */
    const uint32_t* min_member;  /* [n] */
} ks_gangs;
int ks_gang_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const ks_gangs* gangs, int policy,
                 int32_t* out_node_idx, int64_t* out_score, uint32_t* out_placed, uint32_t* out_rounds);

/* ---- asynchronous streaming surface = the reference's Controller queue (src/main.rs:73, :141-148) ----
 * The reference runs reconcile() for many pods concurrently from a work queue.  ks_stream is that queue in front of
 * one snapshot: ks_stream_submit appends pending (unbound) pods and returns at once; a dispatcher thread owned by the
 * library drains everything that has arrived (up to max_batch <= 1024 pods, arrival order) into ONE micro-batch
 * (ks_stream_bind: device-side round loop with capacity commit) and publishes the results; ks_stream_poll collects
 * finished pods without blocking.  Results carry the caller's ticket; node -1 = ReconcileError::NoNodeFound
 * (src/main.rs:116-118).  Pods with spec.nodeName set must be filtered out before submission (src/main.rs:74-76).
 * While a stream is open its snapshot must not be mutated by other calls (same rule as the reference's node store
 * being written only by its reflector).  ks_stream_submit checks the requests as ks_stream_bind does: one outside
 * [0, limit] refuses the whole submit with KS_ERR_RANGE and queues none of its pods. */
typedef struct ks_stream ks_stream;
int ks_stream_open(ks_snapshot* s, int policy, uint32_t max_batch, ks_stream** out);
int ks_stream_submit(ks_stream* q, uint64_t n, const int64_t* req_cpu, const int64_t* req_mem, const uint64_t* sel /* [n*W] */,
                     const uint64_t* tickets /* [n] caller ids, returned by poll */);
/* up to `max` finished pods; *out_n = how many were written (0 = nothing finished yet); never blocks */
int ks_stream_poll(ks_stream* q, uint64_t max, uint64_t* out_ticket, int32_t* out_node_idx, int64_t* out_score, uint64_t* out_n);
int ks_stream_flush(ks_stream* q);  /* blocks until every pod submitted so far has a result waiting in poll */
int ks_stream_stats(ks_stream* q, uint64_t* batches, uint64_t* rounds, uint64_t* max_batch_seen);
void ks_stream_close(ks_stream* q); /* stops the dispatcher; unpolled results are dropped */

/* ---- the reference's own selection policy, seeded (src/main.rs:49-71; ATTEMPTS = 5 at :49) ----
 * For every pod: up to `attempts` draws, uniform with replacement over the snapshot's nodes (:56-57); the first
 * draw whose cell is KS_CELL_OK wins (:61-66); none -> -1 (= None -> ReconcileError::NoNodeFound, :70, :116-118)
 * even when a feasible node exists.  The reference draws from thread_rng; here draw k of pod p is
 * splitmix64 step k of a stream whose state starts at KS_SAMPLING_STREAM(seed, p), node = draw % N, so a run is
 * reproducible and replicas agree.  An empty snapshot wastes every attempt (:56,60): -1, 0 cells.
 * Host output arrays; all but out_node_idx may be NULL:
 *   out_node_idx[P]; out_attempts[P] = cells evaluated; out_draw_node[P*attempts] = node of each draw (-1 = not
 *   made); out_draw_code[P*attempts] = that cell's code, i.e. the InvalidNodeReason the reference logs at :62
 *   (0xff = not made).  first_pod_index offsets p in the stream id (pod i of this call is stream
 *   first_pod_index + i), so a sharded or chunked caller reproduces the single-call result. */
#define KS_REFERENCE_ATTEMPTS 5u
#define KS_SAMPLING_STREAM(seed, p) ((uint64_t)(seed) ^ (((uint64_t)(p) + 1ull) * 0xD1B54A32D192ED03ull))
int ks_select_sampling(ks_snapshot* s, const ks_pods* pods, uint32_t attempts, uint64_t seed, uint64_t first_pod_index,
                       int32_t* out_node_idx, uint32_t* out_attempts, int32_t* out_draw_node, uint8_t* out_draw_code);

/* ---- why a pod has no node: per-pod rejection counts (the batched form of the log line at src/main.rs:62) ----
 * For pod p, over the snapshot's N real nodes only (padding never counts):
 *   insufficient_cpu       nodes with req_cpu > free_cpu                   (half of can_pod_fit, src/predicates.rs:42)
 *   insufficient_memory    nodes with req_mem > free_mem                   (the other half)
 *   not_enough_resources   nodes failing either: cell code KS_CELL_NOT_ENOUGH_RESOURCES (fit is checked first, :68-70)
 *   node_selector_mismatch nodes the pod fits whose labels miss a selector pair: KS_CELL_NODE_SELECTOR_MISMATCH (:72-74)
 * so not_enough_resources + node_selector_mismatch + feasible_cnt == N (feasible_cnt as ks_select reports it) and
 * max(cpu, mem) <= not_enough_resources <= cpu + mem.  Precedence is the reference's (fit first); upstream
 * kube-scheduler runs NodeAffinity before NodeResourcesFit and would count a node failing both as a selector miss. */
typedef struct ks_pod_reasons {
    uint32_t insufficient_cpu, insufficient_memory, not_enough_resources, node_selector_mismatch;
} ks_pod_reasons;
/* out[pods->n] in out_space (KS_MEM_HOST / KS_MEM_DEVICE); pods in pods->mem_space.  Returns after completion when
 * out or the pods are in host memory, after enqueue on cuda_stream (NULL = library stream) when both are on the device. */
int ks_explain(ks_snapshot* s, const ks_pods* pods, ks_pod_reasons* out, int32_t out_space, void* cuda_stream);

/* ---- ranked candidates: the k best feasible nodes per pod (fall-backs after a failed Binding POST, extender
 * "prioritize" replies, "why node X and not node Y") ----
 * For pod p and 1 <= k <= KS_TOPK_MAX, row p holds the min(k, feasible_cnt[p]) feasible nodes with the highest score
 * under `policy`, score descending, ties to the lower node index: the total order ks_select uses, so entry 0 of every
 * row is ks_select's node_idx / score for that pod and policy (on either kernel path) and out_feasible_cnt is its
 * feasible_cnt.  Slots past the feasible count hold node -1 and score 0.  Scores are the values ks_select reports
 * (LEFTOVER: (free_cpu-req_cpu)*2^22 + (free_mem-req_mem); LEAST_ALLOCATED, MOST_ALLOCATED: the integer-floor formulas
 * above).  Padding
 * nodes never appear, and nothing is charged: the snapshot is not changed.
 * KS_ERR_RANGE when k = 0 or k > KS_TOPK_MAX; KS_ERR_INVALID for a bad policy or out_space, or a NULL out_node_idx with
 * pods->n > 0.  pods->n = 0 does nothing; an empty snapshot gives every row -1 / 0 and count 0. */
#define KS_TOPK_MAX 32u
/* out_node_idx[P*k] (row-major, required), out_score[P*k] and out_feasible_cnt[P] (may be NULL), all in out_space;
 * pods in pods->mem_space.  Returns after completion when outputs or pods are on the host, after enqueue on
 * cuda_stream (NULL = library stream) when both are on the device - the same rule as ks_explain. */
int ks_select_topk(ks_snapshot* s, const ks_pods* pods, int policy, uint32_t k, int32_t* out_node_idx,
                   int64_t* out_score, uint32_t* out_feasible_cnt, int32_t out_space, void* cuda_stream);

/* ---- priority preemption: for a pod no node accepts, the node and the lower-priority pods to evict (upstream
 * kube-scheduler's PostFilter / DefaultPreemption without PodDisruptionBudgets; spec extension, DESIGN.md 5d) ----
 * Pending pod p has priority pi_p; bound pod b (its bound index b = its position in `bound`) sits on node b.node with
 * request req_b and priority pi_b.  `bound` must be the list that produced the snapshot's free[] (ks_snapshot_set_bound
 * plus later apply_bind / accepted commits).  For p and real node n:
 *   1. n is eligible only if p fails there on resources alone: !fit(p, n) and the selector matches;
 *   2. L = {b on n : pi_b < pi_p} (strictly lower); empty L: not a candidate;
 *   3. avail = free[n] + sum of req_b over L; unless req_p <= avail (both resources, non-strict): not a candidate;
 *   4. reprieve: visit L by priority descending, ties to the lower bound index (the older pod); b is reprieved when p
 *      still fits avail - req_b (then avail -= req_b), else it is a victim; victims are listed in visit order;
 *   5. more than max_victims victims: not a candidate;
 *   6. among the candidates the plan takes the node with, in order, the lowest highest-victim priority, the lowest
 *      sum of (pi_b + 2^31) over the victims, the fewest victims, the lowest node index;
 *   7. a pod with feasible_cnt > 0 (as ks_select reports it) gets no plan: node -1, no victims, 0 candidates.
 * Nothing is charged and the snapshot is not changed: evict the victims, report them (ks_snapshot_set_bound with the
 * shorter list, or ksh_context_pod_deleted), and the pod schedules on its next pass. */
#define KS_PREEMPT_MAX_VICTIMS 128u
typedef struct ks_bound_pods { /* host memory; the list that produced the snapshot's free[] */
    uint64_t n;
    const int32_t* node_idx;
    const int64_t* req_cpu;
    const int64_t* req_mem;
    const int32_t* priority;
} ks_bound_pods;
typedef struct ks_preemption { /* 32 bytes per pod */
    int32_t node_idx;              /* -1 = no plan */
    uint32_t n_victims;
    uint32_t candidates;           /* nodes where eviction within max_victims makes room (0 when feasible_cnt > 0) */
    uint32_t feasible_cnt;         /* as ks_select reports it */
    int32_t max_victim_priority;   /* INT32_MIN without a plan */
    uint32_t reserved;             /* 0 */
    int64_t victim_priority_sum;   /* sum of (priority + 2^31) over the victims; 0 without a plan */
} ks_preemption;
/* out[pods->n] and out_victims[pods->n * max_victims] (bound indices in visit order, -1 past n_victims; may be NULL)
 * in out_space; pod_priority[pods->n] in pods->mem_space.  `bound` is checked as ks_snapshot_set_bound checks it (node
 * range, per-pod request limits) plus one range rule: for every node, the sum of |req_cpu| and the sum of |req_mem|
 * over its bound pods must each be <= 2^62, which keeps free[n] plus any subset of them inside int64 (KS_ERR_RANGE).
 * KS_ERR_RANGE when max_victims is 0 or above KS_PREEMPT_MAX_VICTIMS, or bound->n >= 2^32; KS_ERR_INVALID for a bad
 * out_space, a NULL bound array, or a NULL pod_priority / out with pods->n > 0.  pods->n = 0 does nothing; an empty
 * snapshot gives every pod no plan.  Returns after completion when pods or outputs are on the host, after enqueue on
 * cuda_stream (NULL = library stream) when both are on the device - the rule of ks_explain. */
#define KS_PREEMPT_MAX_ABS_SUM ((int64_t)1 << 62)
int ks_preempt(ks_snapshot* s, const ks_pods* pods, const int32_t* pod_priority, const ks_bound_pods* bound,
               uint32_t max_victims, ks_preemption* out, int32_t* out_victims, int32_t out_space, void* cuda_stream);

/* ---- preemption under the full filter: ks_preempt with the pod count, scalar resources, taints and required node
 * affinity (upstream DefaultPreemption re-running NodeResourcesFit, TaintToleration and NodeAffinity with the victims
 * removed; spec extension, DESIGN.md 5t) ----
 * `group`, `rules` and `res` mean what they mean for ks_fit_bind (below): pod p belongs to group[p] in [-1, n_groups),
 * group -1 tolerates nothing and has no node affinity; res->node_free[r * N + n] is allocatable minus the bound pods'
 * bound_req, res->pod_req[p * R + r] >= 0.  bound_req[b * R + r] (host memory) is bound pod b's request of resource r,
 * >= 0 (1 for the pod-count resource).  The caller keeps these consistent, as ks_preempt requires of free[]: `bound` is
 * the list that produced free[] and node_free is allocatable minus the bound pods' bound_req.  "p fits n" is ks_fit_bind's
 * resource rule: cpu and memory without a zero skip, each r with upstream's (pod_req 0 always fits).  For pod p, real
 * node n:
 *   1. unresolvable: n fails p's selector, carries a hard taint p's group does not tolerate, or fails the group's
 *      required node affinity; no eviction helps and n is never eligible.  out_unresolvable[p] counts these nodes;
 *   2. eligible: n is resolvable and p does not fit n;
 *   3. L = the pods on n with priority strictly below pi_p; empty L: not a candidate.  For every dimension x (cpu,
 *      memory, each r) avail_x = free_x[n] + sum of req_b,x over L; unless p fits avail: not a candidate;
 *   4. reprieve: L in ks_preempt's order (priority descending, ties to the lower bound index); b is reprieved when p
 *      still fits avail - req_b in every dimension (then avail -= req_b), else it is a victim.  Evicting a victim frees
 *      its pod-count 1 like any other request;
 *   5. steps 5-7 of ks_preempt unchanged: more than max_victims victims is no candidate, the 128-bit node order picks the
 *      plan's node, and feasible_cnt - the resolvable nodes p fits with no eviction - above 0 gives no plan.
 * Rows as ks_preemption; out_victims[p * max_victims ..] bound indices in visit order, -1 past n_victims.  Nothing is
 * charged and the snapshot does not change.  rules->weight_* and preferred terms are checked as ks_node_bind checks them
 * and play no part: preemption does not score.
 * Identities:
 *   (Q1) rules NULL and res NULL: out and out_victims are ks_preempt's, bit for bit, and out_unresolvable[p] is the
 *        number of nodes whose labels miss p's selector;
 *   (Q2) an extra resource that copies cpu (pod_req each pod's positive cpu request, node_free free_cpu, bound_req the
 *        bound cpu) changes nothing;
 *   (Q3) feasible_cnt[p] = ks_select's feasible count minus ks_fit_bind's refusal words 0-2 for p bound alone with no
 *        spread or affinity;
 *   (Q4) evict then bind: with a plan's victims removed (node_free raised by their bound_req, free[] by their requests)
 *        the pod passes the full filter on the planned node, and a second call reports feasible_cnt > 0 for it;
 *   (Q5) returning any single victim makes the pod fail the planned node again.
 * Checked on the host before any device work: every check of ks_preempt on `bound` and max_victims (including the
 * 2^62 rule); ks_fit_bind's checks on group (KS_ERR_INVALID for a NULL group with P > 0 or one outside [-1, G),
 * KS_ERR_RANGE for G > KS_SPREAD_BIND_MAX_GROUPS), rules and res; KS_ERR_INVALID for device-space pods, a NULL
 * pod_priority or out (P > 0), or a NULL bound_req with R > 0 and B > 0; KS_ERR_RANGE for a negative bound_req, or for
 * a (r, n) with |node_free[r * N + n]| + the sum of bound_req over n's bound pods above 2^62 (this keeps every sum of
 * the walk inside int64).  pods->n = 0 does nothing; an empty snapshot gives every pod no plan and 0 unresolvable nodes.
 * One H2D copy of the host arrays, the bound list and bound_req copied into the victim index's scratch, then
 * k_node_rules_setup (ks_node_bind's rule words), the victim index with R request columns, the scan over node tiles,
 * the emit, and one D2H copy; the call returns after completion.
 * Out of scope: PodTopologySpread and InterPodAffinity with the victims removed (upstream re-runs them; they are not
 * inputs here); PodDisruptionBudgets, pod start time, preemptionPolicy, nominatedNodeName; preemption for a gang. */
struct ks_node_rules;     /* defined with ks_node_bind below */
struct ks_bind_resources; /* defined with ks_fit_bind below */
int ks_fit_preempt(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                   uint32_t n_groups, const struct ks_node_rules* rules /* or NULL */,
                   const struct ks_bind_resources* res /* or NULL */, const int32_t* pod_priority /* [P] */,
                   const ks_bound_pods* bound, const int64_t* bound_req /* [B * R], NULL when R = 0 */,
                   uint32_t max_victims, ks_preemption* out /* [P] */, int32_t* out_victims /* [P * max_victims] or NULL */,
                   uint32_t* out_unresolvable /* [P] or NULL */);

/* ---- drain simulation: if a node were removed, where would its pods go (cluster-autoscaler's scale-down simulation,
 * Karpenter consolidation, the descheduler; spec extension, DESIGN.md 5f) ----
 * Candidate d is node node_idx[d] (duplicates allowed) and owns pods [offset[d], offset[d+1]) of `pods`, in the caller's
 * order, 0 to KS_DRAIN_MAX_PODS of them (normally the pods bound to that node).  Each candidate is evaluated on its own
 * against the snapshot's current free[]:
 *   1. destinations: every real node except node_idx[d]; with KS_DRAIN_EXCLUDE_CANDIDATES also no node that appears
 *      anywhere in node_idx (cluster-autoscaler's rule when several nodes are checked for removal together);
 *   2. placement: start from a private copy f of free[]; visit the candidate's pods in array order; each takes the argmax
 *      under `policy` over the destinations where it fits f and its selector matches, ties to the lower node index
 *      (ks_select's order and score), and its request is subtracted from f at that node, so later pods of the same
 *      candidate see the earlier moves (other candidates never do);
 *   3. the first pod with no destination stops the candidate: it and every later pod of the candidate get node -1 and
 *      score 0.  out_placed[d] = pods placed before the stop; the candidate is drainable iff that is its pod count (a
 *      candidate without pods is drainable);
 *   4. nothing is charged: free[], the bit-parallel index and the snapshot are unchanged.
 * Upstream places each pod on the first node its filters accept (with a hinting heuristic); here the destination is the
 * library's own argmax.  Filtering pods before the simulation (PodDisruptionBudgets, DaemonSet and mirror pods, local
 * storage, safe-to-evict) is the caller's job, and so is removing several nodes in sequence: commit one candidate's
 * moves and call again.
 * Host-space pods and outputs: out_placed[n] (required when n > 0), out_node_idx[pods->n] (required when pods->n > 0),
 * out_score[pods->n] (may be NULL).  Checked before any device work: KS_ERR_INVALID for a NULL cand or array, offset[0]
 * != 0, decreasing offsets, offset[n] != pods->n, a candidate node outside [0, N) (so an empty snapshot takes no
 * candidate), unknown flags, a bad policy or device-space pods; KS_ERR_RANGE for a candidate with more than
 * KS_DRAIN_MAX_PODS pods or a request outside [0, limit] (as ks_stream_bind: f stays inside [0, free]).  n = 0 does
 * nothing.  A pod whose selector needs a pair no node carries fits nowhere: its candidate stops there.
 * One H2D copy, one round of two kernels per pod position (round r places pod r of every candidate still running), one
 * D2H copy; the rounds are enqueued back to back. */
#define KS_DRAIN_MAX_PODS 1024u
#define KS_DRAIN_EXCLUDE_CANDIDATES 1u
typedef struct ks_drain_candidates { /* host memory */
    uint64_t n;                /* candidates */
    const int32_t* node_idx;   /* [n] */
    const uint64_t* offset;    /* [n+1], offset[0] = 0, offset[n] = pods->n */
} ks_drain_candidates;
int ks_drain_check(ks_snapshot* s, const ks_pods* pods /* host space */, const ks_drain_candidates* cand, int policy,
                   uint32_t flags, uint32_t* out_placed /* [n], required */, int32_t* out_node_idx /* [pods->n] */,
                   int64_t* out_score /* [pods->n], may be NULL */);

/* ---- scale-up estimate: for pods no node accepts, how many new nodes of each node template would place them
 * (cluster-autoscaler's binpacking estimator, Karpenter's instance-type sizing; spec extension, DESIGN.md 5g) ----
 * Template t is one new, empty node of a node group: allocatable A = (alloc_cpu[t], alloc_mem[t]), capacity
 * F = (free_cpu[t], free_mem[t]) of an empty node (allocatable minus its DaemonSet and system pods), label words
 * labels[t * label_words ...] and max_nodes[t], the nodes the group may still add.  Each template is evaluated on its
 * own; it reads neither the snapshot's node table nor the other templates of the call:
 *   1. eligible: pod p is eligible for t iff its cell code against an empty node of t is KS_CELL_OK (req <= F on both
 *      resources, and (sel & ~labels) == 0 on every word);
 *   2. order: eligible pods by req_cpu/A_c + req_mem/A_m descending (the requests as fractions of the allocatable),
 *      then by lower pod index; compared exactly on the integer key req_cpu*A_m + req_mem*A_c (up to 72 bits);
 *   3. first fit: the open-node list starts empty; each pod, in that order, goes to the lowest-ordinal open node whose
 *      remaining capacity holds it on both resources (non-strict).  If none does and fewer than max_nodes[t] are open,
 *      a new node with remaining F is opened and takes the pod.  Otherwise the pod is not placed and the walk goes on
 *      (a later, smaller pod may still fit).  Placing a pod subtracts its request from its node's remaining capacity;
 *   4. out[t]: nodes opened, pods placed, pods eligible, used_cpu / used_mem = the sum of the placed requests, and
 *      utilization = (used_cpu*100/(nodes*A_c) + used_mem*100/(nodes*A_m))/2 in truncating int64 division (0 when
 *      nodes = 0), in the style of KS_SCORE_LEAST_ALLOCATED;
 *   5. *out_best: the template with the most pods placed, then the highest utilization, then the fewest nodes, then the
 *      lowest index; -1 when no template places a pod.  Other expanders (least-waste, priority, ...) are the caller's
 *      choice: the rows carry what they need;
 *   6. out_node[t * pods->n + p] (may be NULL): the ordinal of the new node of t that p lands on, or -1;
 *      out_reasons[p] (may be NULL): ks_explain's counts with the templates as the nodes, so not_enough_resources +
 *      node_selector_mismatch + (templates p is eligible for) = n - why a pod triggers no scale-up;
 *   7. nothing is charged: free[], the bit-parallel index and the snapshot are unchanged.
 * The label words belong to the call, not to the snapshot's dictionary (a template normally carries pairs no existing
 * node carries yet, such as its instance type); label_words may differ from the snapshot's.  Splitting the templates
 * of one call over several calls gives the same rows; only the best has to be picked again.
 * Checked on the host before any device work: KS_ERR_INVALID for a NULL argument or array, device-space pods, or
 * label_words outside {1, 2, 4, 8}; KS_ERR_RANGE for pods->n > KS_SCALEUP_MAX_PODS, n > KS_SCALEUP_MAX_TEMPLATES, an
 * allocatable outside [1, limit >> 10] (cpu <= 2^26 m, memory <= 2^45 B), a capacity outside [-(limit >> 10), A],
 * max_nodes > KS_SCALEUP_MAX_NODES, or a request outside [0, limit] (as ks_stream_bind).  These keep every sum of a
 * template (at most 1024 nodes of 2^45 B) and the utilization products inside int64.  n = 0 or pods->n = 0 needs no
 * device work: rows and reasons are zero and *out_best = -1.
 * Host-space pods and outputs.  One H2D copy, two kernels (the per-pod reasons only when out_reasons is set), one D2H
 * copy; the best template is picked on the host.  With out_node the snapshot's pinned staging block and its device
 * result block each grow to n * pods->n * 4 bytes (1 GiB each at 4096 templates x 65536 pods) and are kept for reuse
 * until ks_snapshot_destroy.  ks_gang_bind, ks_drain_check and ks_stream_bind stage through the same blocks, and every
 * call that returns only after its host-space results are back stages through the same device blocks, so the snapshot
 * holds the largest any of these calls needed, not their sum.  Callers near the limits who want that memory
 * back can split the templates over calls or use a snapshot of their own for the estimate. */
#define KS_SCALEUP_MAX_NODES 1024u
#define KS_SCALEUP_MAX_PODS 65536u
#define KS_SCALEUP_MAX_TEMPLATES 4096u
typedef struct ks_node_templates { /* host memory */
    uint64_t n;                  /* templates */
    uint32_t label_words;        /* pods->sel is [pods->n * label_words] for this call */
    const int64_t* alloc_cpu;    /* [n] */
    const int64_t* alloc_mem;    /* [n] */
    const int64_t* free_cpu;     /* [n] */
    const int64_t* free_mem;     /* [n] */
    const uint64_t* labels;      /* [n * label_words] */
    const uint32_t* max_nodes;   /* [n] */
} ks_node_templates;
typedef struct ks_scaleup_option { /* 32 bytes per template */
    uint32_t nodes, placed, eligible;
    int32_t utilization;
    int64_t used_cpu, used_mem;
} ks_scaleup_option;
int ks_scaleup_estimate(ks_snapshot* s, const ks_pods* pods /* host space */, const ks_node_templates* t,
                        ks_scaleup_option* out /* [n], required */, int32_t* out_best /* required */,
                        int32_t* out_node /* [n * pods->n] or NULL */, ks_pod_reasons* out_reasons /* [pods->n] or NULL */);

/* ---- replica placement: where R copies of one pod spec land one after another, and how many copies the cluster holds
 * (a Deployment, ReplicaSet or Job scaled out; kubernetes-sigs/cluster-capacity; spec extension, DESIGN.md 5h) ----
 * Spec t is row t of `specs` with replicas[t] copies requested.  Each spec is evaluated on its own against the
 * snapshot's current free[]; nothing is charged.  s_n(j) is the score ks_select reports for the spec on node n with j
 * earlier copies bound there (free minus j * request), under `policy`:
 *   1. c_n, the copies node n takes on its own: 0 unless copy 0's cell code is KS_CELL_OK, else the largest c with
 *      c * req_cpu <= free_cpu and c * req_mem <= free_mem (unbounded when both requests are 0);
 *   2. placement: copy r goes to the node with the highest s_n(j) among the nodes with j < c_n copies placed so far, ties
 *      to the lower node index: ks_select run once per copy with the earlier copies bound.  placed = min(replicas[t],
 *      sum of c_n).  Requests are >= 0, so under LEFTOVER and LEAST_ALLOCATED every s_n(j) is non-increasing in j and
 *      the plan is the first `placed' of all (node, copy) pairs ordered by score descending, node ascending, copy
 *      ascending.  Under MOST_ALLOCATED every s_n(j) is non-decreasing in j: the node being filled never loses to a node
 *      not yet touched, so the plan fills the nodes one after another in order of s_n(0) descending, node ascending,
 *      each with up to c_n copies, and the copies of one node are contiguous in placement order.  Under LEAST_BALANCED
 *      s_n(j) can rise or fall with j: the copies are placed one at a time, exactly as defined;
 *   3. out[t]: capacity = sum of c_n (saturating: UINT64_MAX also means unbounded), placed, nodes = distinct nodes among
 *      the placed copies, feasible_cnt = nodes with c_n >= 1 (ks_select's feasible_cnt), max_per_node = most copies on one
 *      node, last_score = score of copy placed - 1 (0 when nothing is placed);
 *   4. out_node[off_t + r] / out_score[off_t + r], off_t = replicas[0] + ... + replicas[t-1]: node and score of copy r in
 *      placement order; -1 / 0 past `placed'.  Either may be NULL; with both NULL no copy is ordered (the capacity query).
 * To bind one spec's plan, pass its out_node slice to ks_snapshot_commit_claims with the spec's request: every claim is
 * accepted, by construction, and free[] ends as after ks_gang_bind with one singleton group per copy.
 * Checked on the host before any device work: KS_ERR_INVALID for a NULL argument or array, out NULL with specs->n > 0,
 * device-space specs or a bad policy; KS_ERR_RANGE for specs->n > KS_REPLICAS_MAX_SPECS, a replicas[t] above
 * KS_REPLICAS_MAX, a sum of replicas above KS_REPLICAS_MAX_TOTAL or a request outside [0, limit] (as ks_stream_bind: the
 * scores are then monotone and stay inside int64).  replicas[t] = 0 fills the row and places nothing; specs->n = 0 does
 * nothing; an empty snapshot gives capacity 0 and every copy -1.
 * Host-space specs and outputs.  One H2D copy, a fixed sequence of kernels enqueued back to back whose number does not
 * depend on the replicas (a scan, thirteen threshold-search passes of two kernels, the tie split and, with a copy list, one
 * sorting CTA per spec), one D2H copy.  Staging: the snapshot's pinned block and its device input and result blocks hold
 * the specs and n * 32 bytes of rows, plus 12 bytes per requested copy with a copy list (up to 192 MiB at
 * KS_REPLICAS_MAX_TOTAL); its device scratch block holds the search state, plus 20 bytes per requested copy with a copy
 * list (up to 320 MiB).  Like every staging block these grow to the largest call and are kept until
 * ks_snapshot_destroy; ks_gang_bind, ks_drain_check, ks_stream_bind and ks_scaleup_estimate share them.
 * KS_SCORE_LEAST_BALANCED: the scan, then one CTA per spec (specs strided over at most 2 per SM) places that spec's copies
 * one after another, so the time grows with the copies of the largest spec (about 4 us per copy on an H100, DESIGN.md
 * 5j) and no fixed number of passes holds.  Its device scratch block also holds 12 bytes per node for each of those
 * CTAs, as many CTAs as fit in 64 MiB (at least one). */
#define KS_REPLICAS_MAX_SPECS 4096u
#define KS_REPLICAS_MAX 65536u
#define KS_REPLICAS_MAX_TOTAL (1u << 24)
typedef struct ks_replica_plan { /* 32 bytes per spec */
    uint64_t capacity;           /* sum of c_n, saturating; UINT64_MAX also = unbounded */
    uint32_t placed;
    uint32_t nodes;              /* distinct nodes among the placed copies */
    uint32_t feasible_cnt;       /* nodes with c_n >= 1 = ks_select's feasible_cnt */
    uint32_t max_per_node;       /* most copies placed on one node */
    int64_t last_score;          /* score of copy placed-1; 0 when placed = 0 */
} ks_replica_plan;
int ks_place_replicas(ks_snapshot* s, const ks_pods* specs /* host space */, const uint32_t* replicas /* [specs->n] */,
                      int policy, ks_replica_plan* out /* [specs->n] */, int32_t* out_node /* [sum replicas] or NULL */,
                      int64_t* out_score /* [sum replicas] or NULL */);

/* ---- topology spread for replica placement: where R copies of a pod spec land under a zone or hostname maxSkew, and
 * how many fit (upstream PodTopologySpread, whenUnsatisfiable: DoNotSchedule; spec extension, DESIGN.md 5k) ----
 * One constraint per spec whose label selector matches the spec's own pods (the copies count themselves), with
 * nodeAffinityPolicy: Honor, nodeTaintsPolicy: Ignore and minDomains.  Domains are dense ids 0..D-1 of one topology key;
 * node_domain[n] = -1 means node n lacks the key.  For spec t:
 *   1. node n is eligible when node_domain[n] >= 0 and the spec's selector matches it ((sel & ~labels) == 0 on every
 *      word); resource fit plays no part.  E_t = the domains that hold an eligible node;
 *   2. cnt[d] starts at existing[t * D + d], the pods already bound in domain d that match the constraint's selector
 *      (existing NULL: zeros);
 *   3. m = min of cnt[d] over E_t, or 0 when |E_t| < min_domains[t] (upstream's minDomains rule).  E_t empty: nothing
 *      is placed;
 *   4. copy r goes to the node with the highest s_n(j_n) among the eligible nodes with j_n < c_n (j_n = copies already
 *      on n; c_n and s_n(j) exactly as ks_place_replicas defines them) and cnt[d(n)] + 1 - m <= max_skew[t]; ties to
 *      the lower node index.  Then j_n, cnt[d(n)] and m are updated.  The first copy with no candidate stops the spec
 *      (nothing changes after a stop, so no later copy could be placed): the rest get node -1 and score 0;
 *   5. out[t]: placed, nodes, max_per_node and last_score as in ks_replica_plan; eligible_domains = |E_t|; min_count = m
 *      after the last copy; blocked_domain = the lowest domain of E_t that the skew rule still admits but whose eligible
 *      nodes hold no further copy, -1 when every copy was placed or no such domain exists (E_t empty, or minDomains held
 *      m at 0 and every domain is at max_skew).  When m is a true minimum, every domain at m is then full, so this is
 *      the domain that blocks the scale-out;
 *   6. out_node / out_score as in ks_place_replicas (per-spec offset = prefix sum of replicas), out_domain_count[t * D +
 *      d] = the final cnt[d].  Each may be NULL;
 *   7. nothing is charged; committing a spec's out_node slice with ks_snapshot_commit_claims accepts every claim.
 * If every node has a domain and max_skew >= replicas + max(existing), or all nodes share one domain, the plan is
 * ks_place_replicas' plan.  With node_domain[n] = n (kubernetes.io/hostname), max_skew 1 and no existing pods, the copies
 * go to distinct nodes in order of copy 0's score until every node with room holds one.
 * Limits and checks as ks_place_replicas (specs, replicas per spec and in total, requests in [0, limit]; every policy),
 * plus, on the host before any device work: KS_ERR_INVALID for a NULL spread, node_domain or max_skew, or a node_domain
 * entry outside [-1, D); KS_ERR_RANGE for D = 0 or D > KS_SPREAD_MAX_DOMAINS, a max_skew of 0, an existing entry above
 * KS_SPREAD_MAX_EXISTING, or T * D > KS_SPREAD_MAX_COUNTS when existing or out_domain_count is given.  An empty
 * snapshot gives every row zeros with blocked_domain = -1, every copy -1, and counts = existing.
 * Host-space arguments and outputs.  One H2D copy; one kernel orders the nodes by domain (a stable sort, once per call);
 * then one CTA per spec (specs strided over at most 2 per SM) places that spec's copies one after another, so the time
 * grows with the copies of the largest spec, as KS_SCORE_LEAST_BALANCED's ks_place_replicas; one D2H copy.  Staging: the
 * snapshot's pinned block and its device input and result blocks hold the specs, 4 bytes per node, 4 * T * D bytes of
 * existing counts when given, n * 32 bytes of rows, 12 bytes per requested copy with a copy list and 4 * T * D bytes of
 * counts when asked; its device scratch block holds 16 bytes per node for the order, and per CTA 12 bytes per node,
 * 20 bytes per domain and 12 bytes per 1024-node block, as many CTAs as fit in 64 MiB (at least one).  The blocks are
 * shared with the other staged calls and grow to the largest. */
#define KS_SPREAD_MAX_DOMAINS (1u << 20)
#define KS_SPREAD_MAX_EXISTING (1u << 24)
#define KS_SPREAD_MAX_COUNTS (1ull << 26)
typedef struct ks_spread {          /* host memory */
    uint32_t n_domains;             /* D >= 1 */
    const int32_t* node_domain;     /* [N], each in [-1, D) */
    const uint32_t* max_skew;       /* [T], >= 1 */
    const uint32_t* min_domains;    /* [T] or NULL (= no minDomains) */
    const uint32_t* existing;       /* [T * D] or NULL (= 0) */
} ks_spread;
typedef struct ks_spread_plan {     /* 32 bytes per spec */
    uint32_t placed;
    uint32_t nodes;                 /* distinct nodes among the placed copies */
    uint32_t max_per_node;          /* most copies placed on one node */
    uint32_t eligible_domains;      /* |E_t| */
    uint32_t min_count;             /* m after the last copy */
    int32_t blocked_domain;         /* see 5 above; -1 = none */
    int64_t last_score;             /* score of copy placed-1; 0 when placed = 0 */
} ks_spread_plan;
int ks_place_replicas_spread(ks_snapshot* s, const ks_pods* specs /* host space */, const uint32_t* replicas /* [n] */,
                             const ks_spread* spread, int policy, ks_spread_plan* out /* [specs->n] */,
                             int32_t* out_node /* [sum replicas] or NULL */, int64_t* out_score /* [sum replicas] or NULL */,
                             uint32_t* out_domain_count /* [specs->n * D] or NULL */);

/* ---- topology spread over several keys: the same placement when every spec carries one constraint per topology key,
 * such as topology.kubernetes.io/zone and kubernetes.io/hostname together (upstream: a node must pass every constraint
 * the pod carries; DESIGN.md 5l) ----
 * K = n_keys keys, 1 <= K <= KS_SPREAD_MAX_KEYS.  Key k has D_k = n_domains[k] dense domains and its own
 * node_domain[k][N] (-1 = node lacks the key).  Spec t carries one constraint per key: max_skew[t * K + k] >= 1,
 * min_domains[t * K + k] and existing counts.  Specs with different key sets go in different calls.  S = sum of D_k,
 * P_k = D_0 + ... + D_{k-1}.  For spec t:
 *   1. node n is eligible when node_domain[k][n] >= 0 for every k and the spec's selector matches it (nodes without all
 *      the keys are neither counted nor chosen); resource fit plays no part.  E_{t,k} = the key-k domains that hold an
 *      eligible node;
 *   2. cnt_k[d] starts at existing[t * S + P_k + d] (existing NULL: zeros);
 *   3. m_k = min of cnt_k over E_{t,k}, or 0 when |E_{t,k}| < min_domains[t * K + k].  No eligible node: nothing is placed;
 *   4. copy r goes to the eligible node with j_n < c_n and the highest s_n(j_n) such that, for every k,
 *      cnt_k[d_k(n)] + 1 - m_k <= max_skew[t * K + k]; ties to the lower node index (c_n and s_n(j) as ks_place_replicas
 *      defines them, every policy).  Then j_n, every cnt_k[d_k(n)] and every m_k are updated.  The first copy with no
 *      candidate stops the spec; the rest get node -1 and score 0;
 *   5. out[t * K + k] is a ks_spread_plan: placed, nodes, max_per_node and last_score describe spec t and are the same
 *      in all K of its rows; eligible_domains = |E_{t,k}|; min_count = m_k after the last copy; blocked_domain = the
 *      lowest domain of E_{t,k} that key k's own rule still admits and that holds no eligible node with room (j_n < c_n)
 *      admitted by every other constraint: the lowest domain of key k where capacity and the other keys, not k's own
 *      rule, stop the copies.  -1 when every copy was placed or no such domain exists;
 *   6. out_node / out_score as in ks_place_replicas; out_domain_count[t * S + P_k + d] = the final cnt_k[d].  Each may
 *      be NULL;
 *   7. nothing is charged; committing a spec's out_node slice with ks_snapshot_commit_claims accepts every claim.
 * K = 1 is exactly ks_place_replicas_spread (the same rows, copies and counts).
 * Checks on the host before any device work: those of ks_place_replicas_spread, per key; KS_ERR_INVALID for a NULL
 * spread, max_skew or node_domain[k] with k < K; KS_ERR_RANGE for K outside [1, KS_SPREAD_MAX_KEYS], or T * S >
 * KS_SPREAD_MAX_COUNTS when existing or out_domain_count is given.  An empty snapshot gives every row zeros with
 * blocked_domain = -1, every copy -1, and counts = existing.
 * Host-space arguments and outputs.  One H2D copy; one kernel orders the nodes by domain, one CTA per key; then one CTA
 * per spec places its copies one after another, as ks_place_replicas_spread; one D2H copy.  Staging as
 * ks_place_replicas_spread, with 4 bytes per node and key, 4 * T * S bytes of existing counts and of counts, 32 * T * K
 * bytes of rows; device scratch 16 bytes per node and key for the orders, and per CTA also 8 bytes per secondary domain
 * and 4 per 1024-node block slot of the primary. */
#define KS_SPREAD_MAX_KEYS 4u
typedef struct ks_spread_multi {                      /* host memory */
    uint32_t n_keys;                                  /* K */
    uint32_t n_domains[KS_SPREAD_MAX_KEYS];           /* D_k, k < K */
    const int32_t* node_domain[KS_SPREAD_MAX_KEYS];   /* [N] each, in [-1, D_k) */
    const uint32_t* max_skew;                         /* [T * K], each >= 1 */
    const uint32_t* min_domains;                      /* [T * K] or NULL */
    const uint32_t* existing;                         /* [T * S] or NULL */
} ks_spread_multi;
int ks_place_replicas_spread_multi(ks_snapshot* s, const ks_pods* specs /* host space */,
                                   const uint32_t* replicas /* [n] */, const ks_spread_multi* spread, int policy,
                                   ks_spread_plan* out /* [specs->n * K] */, int32_t* out_node /* [sum replicas] or NULL */,
                                   int64_t* out_score /* [sum replicas] or NULL */,
                                   uint32_t* out_domain_count /* [specs->n * S] or NULL */);

/* ---- topology spread when binding: a mixed pod queue bound one pod at a time, each pod under its own workload's spread
 * constraints (upstream kube-scheduler's one scheduling cycle per pod with PodTopologySpread, whenUnsatisfiable:
 * DoNotSchedule; spec extension, DESIGN.md 5m) ----
 * K = spread->n_keys keys, 1 <= K <= KS_SPREAD_MAX_KEYS, given as in ks_spread_multi: D_k = n_domains[k],
 * node_domain[k][N] (-1 = node lacks the key), S = sum of D_k, P_k = D_0 + ... + D_{k-1}.  G = n_groups groups, one per
 * workload (one constraint set); pod p belongs to group group[p] in [-1, G), -1 = the pod carries no constraint.
 * Group g has max_skew[g * K + k] per key, 0 = g has no constraint on key k (so zone-only, zone + hostname and
 * unconstrained workloads share one queue); C_g = the keys with max_skew >= 1.  min_domains[g * K + k] and
 * existing[g * S + P_k + d] are optional, as in ks_spread_multi with T replaced by G.  Every pod of a group carries the
 * same selector words (KS_ERR_INVALID otherwise), so eligibility is a property of the group.
 *   1. group state, once per call, for every k in C_g: a node is eligible for g when it carries every key of C_g and g's
 *      selector matches it (resource fit plays no part); E_{g,k} = the key-k domains that hold an eligible node;
 *      cnt_{g,k} starts at existing; m_{g,k} = min of cnt_{g,k} over E_{g,k}, or 0 while |E_{g,k}| < min_domains;
 *   2. pods run in array order, one at a time, each against the free[] and counts every earlier pod left.  Pod p's
 *      candidates are the nodes it fits (both resources, non-strict), whose labels its selector matches, and, when
 *      group[p] = g >= 0, that have for every k in C_g a domain d_k(n) >= 0 with cnt_{g,k}[d_k(n)] + 1 - m_{g,k} <=
 *      max_skew[g * K + k].  The pod takes the candidate with the highest score under `policy` (ks_select's score against
 *      the current free[], every policy), ties to the lower node index.  Its request is subtracted from free[n], and for
 *      each k in C_g cnt_{g,k}[d_k(n)] rises by 1 and m_{g,k} is updated.  A pod with no candidate gets node -1 and score
 *      0, and nothing changes.  A pod counts only toward its own group (selectors matching other groups' pods are out
 *      of scope);
 *   3. out_node_idx[P] (required); out_score[P], out_refused[P] and out_domain_count[G * S] may be NULL.  out_refused[p]
 *      = the nodes that passed fit and selector at p's turn but that p's constraints refused (a missing key or the skew),
 *      0 for an unconstrained pod: candidates + refused is the feasible count ks_select would report at that turn.
 *      out_domain_count = the final cnt_{g,k} for k in C_g, existing (or 0) for the keys g does not constrain.
 * free[] is charged, as with ks_gang_bind.  Identities:
 *   (1) every pod in group -1, or every max_skew 0: nodes, scores and the final free[] are those of ks_gang_bind with one
 *       singleton group per pod and min_member 0, under every policy;
 *   (2) one group of R pods with identical requests that constrains every key: its nodes and scores are
 *       ks_place_replicas_spread_multi's copy list for that spec with replicas = R, its counts that call's
 *       out_domain_count, and the final free[] is free[] after ks_snapshot_commit_claims of that list (K = 1: the same
 *       against ks_place_replicas_spread).  A pod that fails changes nothing, so every later identical pod of its group
 *       fails too, which is the plan's stop rule.
 * Checked on the host before any device work and before free[] changes: requests in [0, limit] (as ks_stream_bind,
 * KS_ERR_RANGE); the per-key checks of ks_place_replicas_spread_multi (max_skew 0 allowed here); KS_ERR_INVALID for a
 * group entry outside [-1, G), device-space pods, a bad policy, a NULL spread, group, max_skew (G > 0), node_domain[k] or
 * out_node_idx (P > 0), or unequal selectors within a group; KS_ERR_RANGE for P > KS_SPREAD_BIND_MAX_PODS,
 * G > KS_SPREAD_BIND_MAX_GROUPS or G * S > KS_SPREAD_MAX_COUNTS (the counts live on the device whether or not they are
 * returned).  P = 0 does nothing; an empty snapshot places nothing and returns counts equal to existing.
 * Host-space arguments and outputs.  One H2D copy; one kernel builds the group state (one CTA per group); one cooperative
 * launch walks the pods with two grid barriers per pod, as ks_gang_bind's groups; one D2H copy.  Staging: the snapshot's
 * pinned block and device input and result blocks hold the pods, 4 bytes per pod of groups and of refusals, 4 * K * N
 * bytes of node domains, the groups' selectors and constraints and 4 * G * S bytes of counts; its device scratch block
 * holds G * S bytes of eligible-domain flags and 16 bytes per (group, key). */
#define KS_SPREAD_BIND_MAX_PODS 65536u
#define KS_SPREAD_BIND_MAX_GROUPS 4096u
int ks_spread_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                   uint32_t n_groups, const ks_spread_multi* spread /* max_skew etc. [G * K], existing [G * S] */,
                   int policy, int32_t* out_node_idx /* [P] */, int64_t* out_score /* [P] or NULL */,
                   uint32_t* out_refused /* [P] or NULL */, uint32_t* out_domain_count /* [G * S] or NULL */);

/* ---- inter-pod affinity when binding: ks_spread_bind with required pod affinity and anti-affinity (upstream
 * InterPodAffinity's Filter, requiredDuringSchedulingIgnoredDuringExecution; spec extension, DESIGN.md 5n) ----
 * The arguments of ks_spread_bind, with topo->max_skew allowed NULL (= every max_skew 0, no spread constraint), and a
 * term list aff.  Groups stand for label classes: the caller resolves each term's labelSelector and namespaces into the
 * groups whose pods it matches, so group -1 is a pod that no term matches and that carries no term.  Term t belongs to
 * the pods of group owner[t], is KS_POD_AFFINITY or KS_POD_ANTI_AFFINITY, has topology key key[t] (an index into topo's
 * K keys) and matches the pods of the groups target[target_offset[t] .. target_offset[t + 1]).  The E existing pods are
 * bound pods, pod e of group existing_group[e] on node existing_node[e]; they need to be listed only when some term
 * matches them or they carry terms.  "Bound" below means the existing pods and every earlier pod of this call.  For pod
 * p of group g >= 0 and node n, with d_k(n) = topo->node_domain[k][n]:
 *   1. incoming anti-affinity: n is refused when, for some anti term of g on key k, d_k(n) >= 0 and a bound pod of a
 *      target group sits on a node of domain d_k(n) (a node without key k passes that term);
 *   2. existing anti-affinity (symmetry): n is refused when some bound pod, of group h, carries an anti term on key k
 *      that targets g, d_k(n) >= 0 and that pod sits in domain d_k(n);
 *   3. affinity: with M_g = the groups every affinity term of g targets, n is refused when it lacks the key of some
 *      affinity term of g, or when for some affinity term on key k no bound pod of a group in M_g sits in domain d_k(n).
 *      Upstream's first-pod rule: when no bound pod of M_g sits on a node that carries one of those keys and g is in
 *      M_g, the terms hold on every node that carries their keys;
 *   4. pods run as in ks_spread_bind, one at a time in array order: pod p's candidates are fit, selector and spread
 *      (ks_spread_bind's rule 2, unchanged) and rules 1-3; it takes the best candidate under `policy`, ties to the lower
 *      node index, free[] is charged and the pod is bound.  A pod with no candidate changes nothing;
 *   5. out_refused[2p] = the nodes that passed fit and selector but failed spread (ks_spread_bind's out_refused[p]);
 *      out_refused[2p + 1] = the nodes that passed fit, selector and spread but failed rules 1-3 (upstream's filter
 *      order: PodTopologySpread before InterPodAffinity).  out_node_idx, out_score and out_domain_count as in
 *      ks_spread_bind.
 * Identities:
 *   (I1) n_terms = 0: nodes, scores, out_refused[2p], counts and the final free[] are ks_spread_bind's, and every
 *        out_refused[2p + 1] is 0;
 *   (I2) n_terms = 0 and topo->max_skew NULL: the result is ks_gang_bind's with one singleton group per pod;
 *   (I3) one group of R identical pods, one anti term of the group on itself on a key every node carries, no existing
 *        pods: the nodes and scores are ks_place_replicas_spread's copy list (that key, max_skew 1) up to the first copy
 *        whose domain already holds one; every later pod is unbound;
 *   (I4) "g anti h on key k" and "h anti g on key k" give the same result: anti-affinity is symmetric in its owner.
 * Checked on the host before any device work and before free[] changes: every check of ks_spread_bind (max_skew NULL
 * allowed); KS_ERR_INVALID for an owner, target or existing group outside [0, G), an existing node outside [0, N), a
 * kind other than 0 or 1, a key >= K, decreasing target_offset, or a NULL array that is needed; KS_ERR_RANGE for
 * n_terms > KS_AFFINITY_MAX_TERMS, more than KS_AFFINITY_MAX_TARGETS targets, E > KS_AFFINITY_MAX_EXISTING, compiled
 * counters above KS_SPREAD_MAX_COUNTS words, or update entries above KS_AFFINITY_MAX_UPDATES.  aff NULL = no term and
 * no existing pod.
 * The terms are compiled on the host into per-(group, key) counter arrays (B_{g,k} for rules 1 and 2, A_{g,k} for rule
 * 3, D_k words each) and, per group h, the deduplicated (g, k, B|A) entries that a bind of a pod of h raises; one update
 * entry per (g, k, kind).  Host-space arguments and outputs; one H2D copy; ks_spread_bind's setup kernel and one that
 * applies the existing pods' entries; one cooperative launch that walks the pods (at most 2K counter loads per node);
 * one D2H copy.  The bit-parallel index is marked stale. */
#define KS_POD_AFFINITY 0
#define KS_POD_ANTI_AFFINITY 1
#define KS_AFFINITY_MAX_TERMS 16384u
#define KS_AFFINITY_MAX_TARGETS (1ull << 22)
#define KS_AFFINITY_MAX_EXISTING (1ull << 24)
#define KS_AFFINITY_MAX_UPDATES (1ull << 24)
typedef struct ks_pod_affinity {   /* host memory */
    uint32_t n_terms;              /* T */
    const int32_t* owner;          /* [T] group in [0, G) whose pods carry the term */
    const uint8_t* kind;           /* [T] KS_POD_AFFINITY / KS_POD_ANTI_AFFINITY */
    const uint32_t* key;           /* [T] topology key index in [0, K) of topo's keys */
    const uint64_t* target_offset; /* [T + 1] */
    const int32_t* target;         /* groups whose pods the term's labelSelector + namespaces match */
    uint64_t n_existing;           /* E: bound pods that some term matches or that carry terms */
    const int32_t* existing_group; /* [E] in [0, G) */
    const int32_t* existing_node;  /* [E] in [0, N) */
} ks_pod_affinity;
int ks_affinity_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                     uint32_t n_groups, const ks_spread_multi* topo /* keys; max_skew may be NULL = no spread constraint */,
                     const ks_pod_affinity* aff /* or NULL */, int policy, int32_t* out_node_idx /* [P] */,
                     int64_t* out_score /* [P] or NULL */, uint32_t* out_refused /* [2P] or NULL */,
                     uint32_t* out_domain_count /* [G * S] or NULL */);

/* ---- soft constraints when binding: ks_affinity_bind scored as kube-scheduler's default profile scores, with
 * PodTopologySpread's ScheduleAnyway constraints and InterPodAffinity's preferred terms (upstream scoring.go of both
 * plugins, restated here; spec extension, DESIGN.md 5o) ----
 * The arguments of ks_affinity_bind plus `scoring`.  The queue is bound exactly as ks_affinity_bind binds it - the same
 * candidates (fit, selector, hard spread, rules 1-3), order, charge, refusals and hard counts - except for the score that
 * picks among the candidates.  Term kinds 2 and 3 are preferred terms: they score and never filter.  term_weight[t] is
 * the weight of term t, in [1, 100] for a preferred term and 0 for a required one (NULL = all 0).
 * For pod p of group g at its turn: F = its candidates (ks_affinity_bind's rule 4); Sigma_g = the keys k with
 * soft_skew[g * K + k] >= 1; sc_{g,k}[d] = a soft count per (group, key), starting at topo->existing (or 0).
 * PodTopologySpread (soft).  Sigma_g empty (or g = -1): pts(n) = 0 for every n (upstream's Skip).  Otherwise:
 *   - ignored: when soft_all_keys[g] = 1, a node of F that lacks some key of Sigma_g is ignored;
 *   - size_k, k in Sigma_g: the number of distinct domains d_k(n) >= 0 over the non-ignored nodes of F, plus 1 when
 *     soft_all_keys[g] = 0 and some node of F lacks k (upstream counts the empty label value as a domain);
 *   - w_k = log((double)(size_k + 2)), by the C library's log, on the host, into a table indexed by size;
 *   - raw(n), n not ignored: GoRound( sum over k in Sigma_g with d_k(n) >= 0, in ascending k, of
 *     ((double)sc_{g,k}[d_k(n)] * w_k + (double)(soft_skew[g * K + k] - 1)) ), every IEEE operation rounded on its
 *     own (no FMA contraction); GoRound rounds half away from zero;
 *   - with min and max over the non-ignored nodes of F, max starting at 0: pts(n) = 0 for an ignored node, else 100
 *     when max = 0, else 100 * (max + min - raw(n)) / max in int64;
 *   - when the pod binds on n, sc_{g,k}[d_k(n)] rises by 1 for each k in Sigma_g with d_k(n) >= 0; when
 *     soft_all_keys[g] = 1, only if n carries every key of Sigma_g.
 * InterPodAffinity (preferred, and the existing pods' required affinity).  For each bound pod b of group h on node m and
 * each key k with d_k(m) >= 0, every node of b's domain of key k gains:
 *   - +w_t for each preferred affinity term of g on key k that targets h, -w_t for each preferred anti-affinity one;
 *   - +hard_affinity_weight for each required affinity term of h on k that targets g, +w_t for each preferred affinity
 *     term of h on k that targets g, -w_t for each preferred anti-affinity one.
 *   Duplicate terms count twice; a term matches a pod once however often its target list names the pod's group.  A
 *   self term (g targets g) counts twice against a bound pod of g: once as the incoming pod's term and once as the
 *   bound pod's.  raw(n) = the sum over the keys n carries (int64, may be negative); with min and max over F,
 *   ipa(n) = max > min ? (int64)(100.0 * ((double)(raw(n) - min) / (double)(max - min))) : 0.
 * Total: score(n) = policy_score(n) + weight_spread * pts(n) + weight_affinity * ipa(n); the pod takes the highest
 * total, ties to the lower node index.  Policies 1, 3 and 4 (upstream's 0-100 scales; 4 is the default profile's
 * resource pair); LEFTOVER's scale would swamp every soft term.
 * Outputs: out_node_idx, out_refused [2P], out_domain_count as ks_affinity_bind; out_score = the total;
 * out_parts[3p .. 3p + 2] = the winner's policy score, pts and ipa (zeros for an unbound pod); out_soft_count = the
 * final sc.  Each but out_node_idx may be NULL.
 * Departures from upstream: ties go to the lowest index instead of at random; w_k comes from libm, not Go's math.Log;
 * size_k is a distinct-domain count for every key, which is upstream's hostname special case whenever hostnames are
 * unique; TaintToleration, NodeAffinity (see ks_node_bind) and ImageLocality are not modelled (constant for pods and nodes without taints
 * or preferences, and the total omits those constants); nodeInclusionPolicies and matchLabelKeys are out of scope.
 * Identities, policies 1, 3 and 4:
 *   (J1) soft_skew NULL, no preferred term and hard_affinity_weight = 0 (or weight_spread = weight_affinity = 0): the
 *        nodes, hard counts, free[] and both refusals are ks_affinity_bind's, out_score is its score and out_parts is
 *        (score, 0, 0);
 *   (J2) soft constraints and preferred terms only on keys where every node shares one domain: every node of F has
 *        pts = 100 (0 if ignored) and ipa = 0; the nodes are ks_affinity_bind's, and each score is higher by exactly
 *        100 * weight_spread when Sigma_g is non-empty;
 *   (J3) for g != h, "g preferred-(anti-)affine to h on k, weight w" and "h preferred-(anti-)affine to g on k, weight
 *        w" give the same result.
 * Checked on the host before any device work and before free[] changes: every check of ks_affinity_bind, with kinds 0
 * to 3; KS_ERR_INVALID for a NULL scoring, a preferred term whose weight is outside [1, 100], a required term with a
 * non-zero weight, a plugin weight or hard_affinity_weight above 100, a soft_all_keys entry above 1, or a policy other
 * than 1, 3 and 4; KS_ERR_RANGE for more than 2^26 IPA counter words or KS_AFFINITY_MAX_UPDATES IPA update entries.
 * The terms compile into int64 counters I_{g,k} (D_k words) per (incoming group, key) with a non-zero coefficient, and
 * per bound group h the entries (g, k, c) that a bind of a pod of h adds to I_{g,k}[d_k(n)], so a node's IPA raw is
 * at most K counter loads.  Host-space arguments and outputs; one H2D copy; ks_affinity_bind's setup kernels and one
 * that applies the existing pods' IPA entries; one cooperative launch with three or four grid barriers per pod; one
 * D2H copy.  The bit-parallel index is marked stale. */
#define KS_POD_AFFINITY_PREFERRED 2      /* scores only; never filters */
#define KS_POD_ANTI_AFFINITY_PREFERRED 3
typedef struct ks_bind_scoring {         /* host memory */
    const uint32_t* soft_skew;           /* [G * K] or NULL: ScheduleAnyway maxSkew of group g on key k, 0 = none */
    const uint8_t* soft_all_keys;        /* [G] or NULL (= all 1): 1 = explicit constraints, 0 = system-defaulted */
    const uint32_t* term_weight;         /* [T] or NULL: weight in [1, 100] of each preferred term, 0 for required ones */
    uint32_t hard_affinity_weight;       /* upstream hardPodAffinityWeight, [0, 100]; upstream default 1 */
    uint32_t weight_spread;              /* PodTopologySpread plugin weight, [0, 100]; default profile 2 */
    uint32_t weight_affinity;            /* InterPodAffinity plugin weight, [0, 100]; default profile 2 */
} ks_bind_scoring;
int ks_profile_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                    uint32_t n_groups, const ks_spread_multi* topo /* keys; max_skew may be NULL */,
                    const ks_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring, int policy,
                    int32_t* out_node_idx /* [P] */, int64_t* out_score /* [P] or NULL */,
                    int64_t* out_parts /* [3P] or NULL */, uint32_t* out_refused /* [2P] or NULL */,
                    uint32_t* out_domain_count /* [G * S] or NULL */, uint32_t* out_soft_count /* [G * S] or NULL */);

/* ---- taints and node affinity when binding: ks_profile_bind with upstream's TaintToleration and NodeAffinity
 * plugins, Filter and Score (restated here; spec extension, DESIGN.md 5p) ----
 * The arguments of ks_profile_bind plus `rules` (host memory).  All pods of one group share its tolerations and node
 * affinity; group -1 tolerates nothing and has no node affinity, and is still filtered by taints.
 * Taints: the caller numbers up to 64 distinct (key, value, effect) triples.  node_taint_hard[n] holds the bits of node
 * n's NoSchedule and NoExecute taints, node_taint_soft[n] those of its PreferNoSchedule taints; tolerate_hard[g] and
 * tolerate_soft[g] the bits group g tolerates (the soft mask from the tolerations whose effect is empty or
 * PreferNoSchedule only, as upstream's getAllTolerationPreferNoSchedule).  Each of the four may be NULL (= all 0).
 * Node affinity, resolved to domain sets: KN = n_keys rule keys, key k with D_k = n_domains[k] domains and
 * node_domain[k][n] in [-1, D_k) (-1 = the node lacks the key), numbered as ksh_context_topology_domains numbers them.
 * Expression x is (expr_key[x], a set over 0..D_k): words [expr_set_offset[x], expr_set_offset[x + 1]) of expr_set,
 * exactly (D_k + 1 + 63) / 64 of them, bit i = domain i, bit D_k = "absent", no bit above D_k.  A node passes the
 * expression iff bit (d >= 0 ? d : D_k) is set.  Term t of group term_owner[t] is the AND of its expressions
 * [term_expr_offset[t], term_expr_offset[t + 1]); a term with no expression matches nothing.  term_weight[t] = 0 makes
 * it a required term (the group's required terms are ORed; a group without one has no required affinity), a weight in
 * [1, 100] a preferred one.  At most KS_NODE_RULES_MAX_PREFERRED preferred terms per group.
 * For pod p of group g and node n, the filters run in this order: fit and selector; taints: refused when
 * node_taint_hard[n] & ~tolerate_hard[g] != 0; required node affinity; hard spread; rules 1-3 of ks_affinity_bind.
 * Spread eligibility (upstream's nodeAffinityPolicy Honor, nodeTaintsPolicy Ignore): a group's eligible domains come
 * from the nodes that pass its selector, its required node affinity and carry its constrained keys; taints do not count.
 * Scores over F, the pod's candidates after every filter:
 *   - TaintToleration: raw(n) = popcount(node_taint_soft[n] & ~tolerate_soft[g]); with max over F, tt(n) = 100 when
 *     max = 0, else 100 - 100 * raw(n) / max in int64 (upstream DefaultNormalizeScore(100, reverse = true));
 *   - NodeAffinity: raw(n) = the sum of the weights of g's preferred terms n matches; na(n) = 0 when max = 0, else
 *     100 * raw(n) / max (DefaultNormalizeScore(100, false)); 0 for a group without preferred terms (upstream's Skip);
 *   - total = ks_profile_bind's total + weight_taint * tt(n) + weight_node_affinity * na(n), ties to the lower index.
 * Outputs as ks_profile_bind's, except: out_parts[5p .. 5p + 4] = (policy, pts, ipa, tt, na) of the winner (zeros for
 * an unbound pod); out_refused[4p .. 4p + 3] = the nodes that fit (fit and selector) but carry an untolerated hard
 * taint, the nodes that fit and are tolerated but fail required node affinity, then ks_profile_bind's two words over
 * the nodes that pass both.
 * Identities, policies 1, 3 and 4:
 *   (K1) rules NULL: every output is ks_profile_bind's, bit for bit, and out_parts words 3 and 4 are 0;
 *   (K2) no node carries a taint and no group has a node-affinity term: the nodes, refusal words 2-3, both counts and
 *        free[] are ks_profile_bind's, refusal words 0-1 are 0 and every score is higher by exactly 100 * weight_taint;
 *   (K3) a required term `key In {v}` binds the same nodes as a nodeSelector key=v on the same groups;
 *   (K4) a NoSchedule taint that every group tolerates changes nothing but the score constant.
 * Checked on the host before any device work and before free[] changes: every check of ks_profile_bind; KS_ERR_INVALID
 * for a taint bit at or above n_taints, a key at or above n_keys, a NULL node_domain or array that is needed, a node
 * domain outside [-1, D_k), a set of the wrong width or with a bit above D_k, decreasing offsets, a term owner outside
 * [0, G), a term weight above 100 or a plugin weight above 100; KS_ERR_RANGE for more than 64 taints, more than
 * KS_NODE_RULES_MAX_KEYS keys, more than KS_NODE_RULES_MAX_PREFERRED preferred terms in a group, or more than
 * KS_NODE_RULES_MAX_WORDS rule words.
 * The groups are mapped to node-rule classes, their distinct (tolerations, terms) signatures; group -1 shares the class
 * of the groups without rules.  k_node_rules_setup writes one 32-bit word per (class, node): the filter reason, the
 * "passes required affinity" bit, the PreferNoSchedule count and the preferred-affinity raw, so the per-pod cycle reads
 * one extra word per node however many expressions a group carries; rule words = classes x N.
 * Out of scope: node rules in ks_select, ks_stream_bind, ks_gang_bind, the planners and ks_explain; matchFields;
 * nodeTaintsPolicy Honor; NodeUnschedulable; ImageLocality; NoExecute eviction and tolerationSeconds; random ties. */
#define KS_NODE_RULES_MAX_TAINTS 64u
#define KS_NODE_RULES_MAX_KEYS 16u
#define KS_NODE_RULES_MAX_PREFERRED 4096u     /* per group: the raw sum stays below 2^22 */
#define KS_NODE_RULES_MAX_WORDS (1ull << 26)  /* classes x nodes */
typedef struct ks_node_rules {                /* host memory */
    uint32_t n_taints;                        /* [0, 64] */
    const uint64_t* node_taint_hard;          /* [N] or NULL */
    const uint64_t* node_taint_soft;          /* [N] or NULL */
    const uint64_t* tolerate_hard;            /* [G] or NULL */
    const uint64_t* tolerate_soft;            /* [G] or NULL */
    uint32_t n_keys;                          /* KN, [0, KS_NODE_RULES_MAX_KEYS] */
    uint32_t n_domains[KS_NODE_RULES_MAX_KEYS];
    const int32_t* node_domain[KS_NODE_RULES_MAX_KEYS]; /* [N] each */
    uint32_t n_exprs;
    const uint32_t* expr_key;                 /* [X] */
    const uint64_t* expr_set_offset;          /* [X + 1], in words of expr_set */
    const uint64_t* expr_set;
    uint32_t n_terms;
    const int32_t* term_owner;                /* [T], in [0, G) */
    const uint32_t* term_weight;              /* [T]: 0 = required, [1, 100] = preferred */
    const uint32_t* term_expr_offset;         /* [T + 1] */
    uint32_t weight_taint;                    /* TaintToleration plugin weight, [0, 100]; default profile 3 */
    uint32_t weight_node_affinity;            /* NodeAffinity plugin weight, [0, 100]; default profile 2 */
} ks_node_rules;
int ks_node_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                 uint32_t n_groups, const ks_spread_multi* topo /* keys; max_skew may be NULL */,
                 const ks_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                 const ks_node_rules* rules /* or NULL */, int policy, int32_t* out_node_idx /* [P] */,
                 int64_t* out_score /* [P] or NULL */, int64_t* out_parts /* [5P] or NULL */,
                 uint32_t* out_refused /* [4P] or NULL */, uint32_t* out_domain_count /* [G * S] or NULL */,
                 uint32_t* out_soft_count /* [G * S] or NULL */);

/* ---- extended resources when binding: ks_node_bind with the rest of upstream's NodeResourcesFit filter, the pod
 * count and every scalar resource a pod requests (restated here; spec extension, DESIGN.md 5r) ----
 * The arguments of ks_node_bind plus `res` (host memory, may be NULL) and out_free.  R = res->n_res resources, each a
 * row of node_free [R * N] (resource r of node n at r * N + n: allocatable minus what the pods already bound there
 * request; any int64, negative included) and a column of pod_req [P * R] (pod p's request of r at p * R + r, >= 0).
 * Resources are what the caller names them: upstream's pod count is a resource whose node_free is allocatable "pods"
 * minus the pods bound there and whose request is 1 for every pod, group -1 included; nvidia.com/gpu, other extended
 * resources, ephemeral-storage and hugepages-* are resources whose requests are the pods' requests.
 * The fit rule (upstream fitsRequest): node n passes resource r for pod p iff pod_req[p * R + r] == 0 or
 * pod_req[p * R + r] <= free_r[n], free_r[n] being r's free amount at p's turn; a zero request is skipped, so a node with
 * negative free_r still takes a pod that does not request r.  The pod count's `len(pods) + 1 > allowed` is `1 > free`.
 * cpu and memory keep ks_select's rule (no zero skip).
 * For pod p of group g and node n, the filters run in this order: cpu, memory and selector; the R resources; taints;
 * required node affinity; hard spread; rules 1-3 of ks_affinity_bind.  Spread eligibility is ks_node_bind's: resources
 * play no part in it, as upstream.  When p binds on n, free_r[n] -= pod_req[p * R + r] for every r, alongside free[];
 * the scores are ks_node_bind's (the default profile scores cpu and memory only).
 * rules NULL: an empty rule set (no taint, no term) with both plugin weights 0, so the total is ks_profile_bind's; out_parts
 * words 3 and 4 are then 0, as ks_node_bind's K1.
 * Outputs as ks_node_bind's, except: out_refused[5p] = the nodes that pass cpu, memory and selector but fail some
 * resource, and out_refused[5p + 1 .. 5p + 4] = ks_node_bind's four words over the nodes that pass every resource;
 * out_free [R * N] (or NULL) = free_r after the call.
 * Identities, policies 1, 3 and 4:
 *   (L1) res NULL: every output is ks_node_bind's, bit for bit, and every out_refused[5p] is 0;
 *   (L2) every request 0: the outputs are L1's, and out_free == node_free, negative entries included;
 *   (L3) always: out_free[r * N + n] == node_free[r * N + n] - the sum of pod_req[p * R + r] over the pods bound on n;
 *   (L4) every node_free at least the queue's total request of its resource: nodes, scores, parts, words 1-4, both counts
 *        and free[] are ks_node_bind's;
 *   (L5) a resource whose request is each pod's cpu request (all positive) and whose node_free is free_cpu changes
 *        nothing.
 * Checked on the host before any device work and before free[] changes: every check of ks_node_bind; KS_ERR_RANGE for
 * R > KS_BIND_MAX_RESOURCES or a negative request; KS_ERR_INVALID for a NULL node_free (R > 0, N > 0) or pod_req
 * (R > 0, P > 0).
 * With rules given, the call makes ks_node_bind's launches; with rules NULL, one more than ks_node_bind (which then runs
 * ks_profile_bind's walk, K1): k_node_rules_setup over the empty rule set.  Each pod's cycle loads one int64 per node
 * for each resource the pod requests.
 * Out of scope: resources in ks_select, ks_stream_bind, ks_gang_bind, the planners and ks_explain; scoring by them;
 * initContainers and pod overhead; ignoredResources. */
#define KS_BIND_MAX_RESOURCES 8u
typedef struct ks_bind_resources {            /* host memory */
    uint32_t n_res;                           /* R in [0, KS_BIND_MAX_RESOURCES] */
    const int64_t* node_free;                 /* [R * N] */
    const int64_t* pod_req;                   /* [P * R], each >= 0 */
} ks_bind_resources;
int ks_fit_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                uint32_t n_groups, const ks_spread_multi* topo /* keys; max_skew may be NULL */,
                const ks_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                const ks_node_rules* rules /* or NULL */, const ks_bind_resources* res /* or NULL */, int policy,
                int32_t* out_node_idx /* [P] */, int64_t* out_score /* [P] or NULL */,
                int64_t* out_parts /* [5P] or NULL */, uint32_t* out_refused /* [5P] or NULL */,
                uint32_t* out_domain_count /* [G * S] or NULL */, uint32_t* out_soft_count /* [G * S] or NULL */,
                int64_t* out_free /* [R * N] or NULL */);

/* ---- gangs when binding: ks_fit_bind with pod groups placed all or nothing (upstream coscheduling's PodGroup
 * minMember under the full filter; spec extension, DESIGN.md 5s) ----
 * The arguments of ks_fit_bind plus `gangs` (ks_gang_bind's struct, host memory) and out_placed.  Gang j is the pods
 * [offset[j], offset[j + 1]) of the queue: offset[0] = 0, offset[n] = P, every gang holds at least one pod and
 * 0 <= min_member[j] <= its size.  A gang's pods may belong to different groups (a launcher and its workers, say); its
 * size is bounded by the queue's KS_SPREAD_BIND_MAX_PODS only (KS_GANG_MAX_SIZE is ks_gang_bind's batch, not this call's).
 *   1. the pods run in queue order with exactly ks_fit_bind's cycle: the same filters, scores, ties, charge and count
 *      updates, each pod against the state every earlier pod left;
 *   2. after a gang's last pod, placed[j] = the number of its pods that bound; when placed[j] >= min_member[j] the gang
 *      commits and its pods keep their bindings;
 *   3. otherwise it rolls back: every pod of the gang gets node -1, score 0 and zero parts, and every piece of state the
 *      gang changed goes back bit for bit to its value before the gang - free[], free_r, the hard counts, the spread
 *      minima, the inter-pod affinity counters and first-pod flags, the soft counts and the IPA counters - so the next
 *      gang sees exactly what this one saw;
 *   4. out_refused[5p .. 5p + 4] keep the words of pod p's own turn, also when its gang rolls back: they say why the
 *      gang came up short;
 *   5. there is no early exit: every pod of a gang runs its cycle, so every output is defined for every pod.
 * out_domain_count, out_soft_count, out_free and free[] are the values after every rollback; out_placed[n] (or NULL) =
 * placed[j] before any rollback.
 * Identities, policies 1, 3 and 4:
 *   (M1) every min_member 0: every output is ks_fit_bind's, bit for bit, and out_placed[j] counts the gang's bound pods;
 *   (M2) singleton gangs with min_member 1: the same as M1;
 *   (M3) with C the pods of the committed gangs in queue order: their nodes, scores, parts and refusal words are those
 *        of ks_fit_bind run on C alone (the same groups and existing pods), and so are the final counts, soft counts,
 *        free_r and free[];
 *   (M4) every gang rolls back: free[], out_free, the counts and the soft counts are the call's inputs, and a ks_select
 *        after the call, on either path, equals one before it.
 * Checked on the host before any device work and before free[] changes: every check of ks_fit_bind; KS_ERR_INVALID for
 * a NULL gangs, offset or min_member (n > 0), offset[0] != 0, decreasing offsets or offset[n] != P; KS_ERR_RANGE for an
 * empty gang or a min_member above its gang's size.
 * ks_fit_bind's launches, with its walk's own instance: the rollback runs in the commit of the gang's last pod, on one
 * CTA, before that pod's last grid barrier, so a gang adds no barrier.  It subtracts what the gang's bound pods added and
 * recomputes each touched group's spread minimum over that key's eligible domains (up to D_k loads per key) and each
 * touched first-pod flag over the group's affinity counters.  The bit-parallel index is marked stale.
 * Out of scope: a search over placements inside a gang (the walk is greedy, as upstream coscheduling and ks_gang_bind:
 * a gang whose first pod takes a zone without room for the rest fails); permit timeouts; preemption for a gang. */
int ks_gang_fit_bind(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                     uint32_t n_groups, const ks_spread_multi* topo /* keys; max_skew may be NULL */,
                     const ks_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                     const ks_node_rules* rules /* or NULL */, const ks_bind_resources* res /* or NULL */,
                     const ks_gangs* gangs, int policy, int32_t* out_node_idx /* [P] */,
                     int64_t* out_score /* [P] or NULL */, int64_t* out_parts /* [5P] or NULL */,
                     uint32_t* out_refused /* [5P] or NULL */, uint32_t* out_domain_count /* [G * S] or NULL */,
                     uint32_t* out_soft_count /* [G * S] or NULL */, int64_t* out_free /* [R * N] or NULL */,
                     uint32_t* out_placed /* [n] or NULL */);

/* ---- drain simulation under the full filter: ks_drain_check with the pod count, scalar resources, taints and required
 * node affinity (cluster-autoscaler's removal simulation and Karpenter's consolidation running the scheduler's filters;
 * spec extension, DESIGN.md 5u) ----
 * ks_drain_check's steps 1-4 (above), changed only where written here.  `group`, `rules` and `res` mean what they mean
 * for ks_fit_bind: pod p belongs to group[p] in [-1, n_groups), group -1 tolerates nothing, has no node affinity and is
 * still filtered by taints; res->node_free[r * N + n] is allocatable minus what the bound pods request there (any
 * int64), res->pod_req[p * R + r] >= 0 what pod p, one of the pods being drained, requests; the pod count is a resource
 * whose request is 1.
 *   1. destinations: ks_drain_check's - every real node but the candidate's own, and with KS_DRAIN_EXCLUDE_CANDIDATES no
 *      candidate's node at all;
 *   2. placement: each candidate starts from private copies f of free[] and f_r of node_free, and visits its pods in
 *      array order.  Pod p may go to destination n when it passes ks_fit_bind's filter there at that point: cpu and
 *      memory against f (no zero skip), the selector, each resource against f_r (upstream's zero skip: a zero request
 *      always fits), no untolerated hard taint, and the group's required node affinity.  Among those it takes the argmax
 *      of `policy`'s score over f, ties to the lower node index, and its requests are subtracted from f and from every
 *      f_r at that node, so later pods of the candidate see the move.  A requested resource fits before it is
 *      subtracted, so f_r never drops below 0 by a move and never overflows;
 *   3. stop, placed and drainable as ks_drain_check: the first pod with no destination stops the candidate, it and every
 *      later pod get node -1 and score 0, out_placed[d] counts the pods placed before it, and the candidate is
 *      drainable iff that is its pod count;
 *   4. nothing is charged: free[], the bit-parallel index and the snapshot are unchanged.
 * out_refused[4d .. 4d + 3] (or NULL) says why a stopped candidate stopped.  The words count the destinations of its
 * stopping pod p = offset[d] + out_placed[d], at p's turn (against f and f_r after the earlier moves): word 0 the nodes
 * that fail cpu, memory or the selector; word 1 those that pass them but fail a resource; word 2 those that pass all of
 * that but carry a hard taint the group does not tolerate; word 3 those that pass all of that but fail required node
 * affinity.  Words 1-3 are ks_fit_bind's refusal words 0-2 in its filter order, and the four sum to the candidate's
 * destination count.  They are all 0 for a drainable candidate.
 * Scores are the resource policy's, as in ks_drain_check; TaintToleration and NodeAffinity do not score here.  This is
 * deliberate: drainability depends only on the filter and on the order of the moves, and (D1) stays exact.
 * rules->weight_* and preferred terms are checked as ks_node_bind checks them and play no part.
 * Identities:
 *   (D1) rules and res NULL (any group): out_placed, out_node_idx and out_score are ks_drain_check's, bit for bit, at
 *        every policy, with and without KS_DRAIN_EXCLUDE_CANDIDATES;
 *   (D2) an extra resource that copies cpu (pod_req each pod's positive cpu request, node_free free_cpu) changes nothing;
 *   (D3) no node carries a taint, no group has a node-affinity term and every node_free is at least the total request of
 *        its resource over every candidate: the outputs are D1's;
 *   (D4) a drainable candidate's moves, replayed one at a time on a copy of the cluster (free[] reduced by the requests,
 *        node_free by pod_req), pass the full filter at every step;
 *   (D5) a stopped candidate's four words sum to its destination count.
 * Checked on the host before any device work: every check of ks_drain_check; ks_fit_bind's checks on group
 * (KS_ERR_INVALID for a NULL group with pods->n > 0 or one outside [-1, G), KS_ERR_RANGE for G >
 * KS_SPREAD_BIND_MAX_GROUPS), rules and res.  n = 0 does nothing.
 * One H2D copy (the pods in round order with their groups and pod_req, the candidates, the excluded column and
 * node_free, and the rules), k_node_rules_setup (ks_node_bind's rule words), one scan and one commit per round enqueued
 * back to back, with out_refused one counting scan after the last round, and one D2H copy; the call returns after
 * completion.
 * Out of scope: PodTopologySpread and InterPodAffinity with the moved pods (upstream re-runs them; they are not inputs
 * here, as in ks_fit_preempt); PodDisruptionBudgets and pod filtering, the caller's job as in ks_drain_check; scoring by
 * TaintToleration and NodeAffinity; NodeUnschedulable other than through its taint; ks_explain under the full filter
 * (the scale-up estimator under it is ks_fit_scaleup_estimate below). */
int ks_fit_drain_check(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                       uint32_t n_groups, const struct ks_node_rules* rules /* or NULL */,
                       const struct ks_bind_resources* res /* or NULL */, const ks_drain_candidates* cand, int policy,
                       uint32_t flags, uint32_t* out_placed /* [n] */, int32_t* out_node_idx /* [P] */,
                       int64_t* out_score /* [P] or NULL */, uint32_t* out_refused /* [4n] or NULL */);

/* ---- scale-up estimate under the full filter: ks_scaleup_estimate with the pod count, scalar resources, taints and
 * required node affinity on the new nodes (cluster-autoscaler's binpacking estimator and Karpenter's instance-type
 * sizing running the scheduler's filters against a template node; spec extension, DESIGN.md 5v) ----
 * ks_scaleup_estimate's steps 1-7 (above), changed only where written here.  The templates play the part of the nodes
 * in `group`, `rules` and `res`, which mean what they mean for ks_fit_bind with N = T: rules->node_taint_hard/soft[t]
 * and rules->node_domain[k][t] are template t's; group -1 tolerates nothing and has no node affinity;
 * res->node_free[r * T + t] is the amount of resource r on one empty node of template t (its allocatable minus its
 * DaemonSet pods' requests; for the pod count, minus their number; any value in [-2^52, 2^52]) and
 * res->pod_req[p * R + r] >= 0 pod p's request.
 *   1. eligible: pod p is eligible for t iff it passes ks_fit_bind's filter on an empty node of t: cpu and memory <= F
 *      (no zero skip) and the selector; each resource with upstream's zero skip (pod_req == 0 or pod_req <= node_free);
 *      no hard taint of t that p's group does not tolerate; the group's required node affinity;
 *   2. order: unchanged (the cpu/memory key; cluster-autoscaler's decreasing-size orderer scores cpu and memory only);
 *   3. first fit: each open node keeps a remaining amount of every resource, starting from node_free[r * T + t]; a pod
 *      fits an open node when cpu, memory and every resource it requests (zero skip) fit the node's remaining amounts,
 *      and placing it subtracts all its requests.  Opening a node, max_nodes and skipping a pod that fits nowhere are
 *      unchanged;
 *   4. out[t] and *out_best as ks_scaleup_estimate's (utilization over cpu and memory); out_used[t * R + r] (may be
 *      NULL) = the sum of resource r over t's placed pods, so a caller can weigh GPU waste between groups;
 *   5. out_refused[4p .. 4p + 3] (may be NULL) count the templates by the first filter each fails, in ks_fit_bind's
 *      order: word 0 cpu, memory or the selector; word 1 a resource; word 2 an untolerated hard taint; word 3 required
 *      node affinity.  With the templates p is eligible for they sum to T (ks_fit_drain_check's word layout);
 *   6. nothing is charged: free[], the bit-parallel index and the snapshot are unchanged.  rules->weight_* and preferred
 *      terms are checked as ks_node_bind checks them and play no part.
 * Identities:
 *   (E1) rules and res NULL (any groups): out, *out_best and out_node are ks_scaleup_estimate's, bit for bit; out_refused
 *        word 0 is its not_enough_resources + node_selector_mismatch and words 1-3 are 0;
 *   (E2) an extra resource that copies cpu (pod_req each pod's positive cpu request, node_free the template's cpu
 *        capacity F) changes nothing;
 *   (E3) no template carries a taint, no group has a node-affinity term and every node_free is at least the queue's
 *        total request of its resource: rows, best and nodes are E1's;
 *   (E4) replaying each template's out_node, every opened node's summed requests fit F and every node_free in every
 *        dimension (zero skip), and every placed pod is eligible;
 *   (E5) for every pod, the four refusal words plus its eligible-template count equal T;
 *   (E6) splitting the templates over calls gives the same rows, as for ks_scaleup_estimate.
 * Checked on the host before any device work: every check of ks_scaleup_estimate; ks_fit_bind's checks on group
 * (KS_ERR_INVALID for a NULL group with pods->n > 0 or one outside [-1, G), KS_ERR_RANGE for G >
 * KS_SPREAD_BIND_MAX_GROUPS), rules (with N = T) and res; KS_ERR_RANGE for a node_free outside [-2^52, 2^52], which with
 * at most KS_SCALEUP_MAX_NODES nodes per template keeps every per-node remainder and every out_used sum inside int64.
 * n = 0 or pods->n = 0 needs no device work: rows, words and sums are zero and *out_best = -1.
 * One H2D copy (pods, groups, pod_req, templates, node_free, rules), k_node_rules_setup over the templates, one packing
 * kernel, with out_refused one reasons kernel, and one D2H copy; the best template is picked on the host.
 * Out of scope: PodTopologySpread and InterPodAffinity on the new nodes; startup and ignored taints (the caller passes
 * the taints it wants counted); cluster-autoscaler's "last node first" fit heuristic and other expanders; existing
 * nodes (run a bind call first, as in 5g, and pass the pods it leaves unplaced). */
int ks_fit_scaleup_estimate(ks_snapshot* s, const ks_pods* pods /* host space */, const int32_t* group /* [P] */,
                            uint32_t n_groups, const struct ks_node_rules* rules /* node arrays over templates, or NULL */,
                            const struct ks_bind_resources* res /* node_free [R * T], or NULL */,
                            const ks_node_templates* t, ks_scaleup_option* out /* [T] */, int32_t* out_best,
                            int32_t* out_node /* [T * P] or NULL */, uint32_t* out_refused /* [4P] or NULL */,
                            int64_t* out_used /* [T * R] or NULL */);

#ifdef __cplusplus
}
#endif
#endif /* KSCHED_H */
