// ks_launch.h — host-callable launchers implemented in ks_direct.cu / ks_bitpar.cu
#pragma once
#include "ks_internal.cuh"

namespace ks {

cudaError_t launch_free_reduce(int64_t* free_cpu, int64_t* free_mem, const int32_t* bnode, const int64_t* bcpu,
                               const int64_t* bmem, uint64_t B, cudaStream_t st);
cudaError_t launch_node_prio(const int64_t* free_cpu, const int64_t* free_mem, int64_t* prio, uint32_t N,
                             uint32_t Npad, int* range_flag, cudaStream_t st);
cudaError_t launch_check_cells(const NodeTable& nt, const PodView& pv, uint8_t* codes, uint32_t node_begin,
                               uint32_t node_count, cudaStream_t st);
cudaError_t launch_select_sampling(const NodeTable& nt, const PodView& pv, uint32_t attempts, uint64_t seed,
                                   uint64_t pod_offset, int32_t* node_idx, uint32_t* n_attempts, int32_t* draw_node,
                                   uint8_t* draw_code, cudaStream_t st);
// multi-GPU exchange helpers (ks_direct.cu): push finished bindings to the peers (per-cell path), wait for all ranks
cudaError_t launch_exchange_push(const PeerOut& po, const int32_t* node_idx, const int64_t* score, uint32_t P, cudaStream_t st);
cudaError_t launch_exchange_wait(const PeerOut& po, int* error_flag, cudaStream_t st);
cudaError_t launch_fill256(void* dst, uint64_t bytes, uint32_t v, int sms, cudaStream_t st);
// launch geometry of the per-cell kernels (K2d, K2e) for P > 0 pods and Npad > 0 nodes: CTAs over the pods times node
// chunks over gridDim.y; n_chunks > 1 needs partial buffers of n_chunks * P entries (K2d)
struct DirectGrid {
    uint32_t pod_ctas, n_chunks, tiles_per_chunk;
};
DirectGrid direct_grid(uint32_t W, uint32_t P, uint32_t Npad, int sms);
cudaError_t prepare_direct(); // once per snapshot, outside any stream capture
cudaError_t launch_select_direct(const SelectLaunch& L, const PartialView& part, const DirectGrid& g);
// per-pod rejection counts (ks_explain): out = uint32 [P][4] in ks_pod_reasons order, device memory
cudaError_t launch_explain_counts(const NodeTable& nt, const PodView& pv, uint32_t* out, int sms, cudaStream_t st);
// ranked candidates (ks_select_topk): ov.node_idx / score = [P][k], ov.cnt = [P] (score and cnt may be null), device
// memory; with g.n_chunks > 1, part holds g.n_chunks * P * k keys and indices and g.n_chunks * P counts
cudaError_t launch_select_topk(const NodeTable& nt, const PodView& pv, int policy, uint32_t k, const OutView& ov,
                               const PartialView& part, const DirectGrid& g, cudaStream_t st);

// priority preemption (ks_preempt).  The victim index: the bound list sorted by (node, priority ascending), ties by
// descending bound index, so that walking a node's segment backwards visits priority descending, ties to the lower
// bound index.  Device memory, B bound pods, N nodes.
struct VictimIndex {
    const uint32_t* off;     // [N+1]: node n's segment is [off[n], off[n+1])
    const int32_t* min_prio; // [N]: lowest priority on node n, INT32_MAX when it has no pod
    const int32_t* prio;     // [B] sorted
    const int64_t* cpu;      // [B] requests, sorted
    const int64_t* mem;
    const int64_t* pre_cpu;  // [B] inclusive prefix sums of the requests within each segment
    const int64_t* pre_mem;
    const uint32_t* idx;     // [B] bound index
};
struct BoundUpload { // where the host list is copied before build_victim_index
    int32_t* node;
    int64_t* cpu;
    int64_t* mem;
    int32_t* prio;
};
size_t victim_index_bytes(uint64_t B, uint32_t N); // one scratch block holds the upload, the sort and the index
BoundUpload victim_index_inputs(void* scratch, uint64_t B, uint32_t N);
cudaError_t build_victim_index(void* scratch, uint64_t B, uint32_t N, VictimIndex* vx, cudaStream_t st);
// per-(node chunk, pod) results of the scan, [n_chunks][P]
struct PreemptPartials {
    uint64_t* hi; // best candidate key (preempt_key), PREEMPT_NONE when none
    uint64_t* lo;
    uint32_t* cand; // candidate nodes
    uint32_t* cnt;  // feasible nodes
};
// out[P] and victims[P * max_victims] (may be null), device memory.  With nt.N == 0 only the rows are written (no plan).
cudaError_t launch_preempt(const NodeTable& nt, const PodView& pv, const int32_t* pod_prio, const VictimIndex& vx,
                           uint32_t max_victims, const PreemptPartials& part, const DirectGrid& g, ks_preemption* out,
                           int32_t* victims, cudaStream_t st);

// preemption under the full filter (ks_fit_preempt).  The victim index of build_victim_index plus R request columns in
// its sorted order and their per-segment inclusive prefix sums, and what the scan reads beyond ks_preempt's inputs: each
// pod's requests and node-rule class, the free amounts and the rule words of ks_node_bind.  Device memory.
struct FitPreemptArgs {
    uint32_t R;                // [0, KS_BIND_MAX_RESOURCES]
    uint32_t B;                // bound pods
    const int64_t* req;        // [P * R]: pod p's request of r at p * R + r
    const int64_t* node_free;  // [R * N]
    const int32_t* group;      // [P], each in [-1, G)
    const uint32_t* ncls;      // [G + 1]: the class of group g at g + 1, of group -1 at 0
    const uint32_t* nrules;    // [C * N], written by k_node_rules_setup
    const int64_t* vres;       // [R * B]: bound requests in the victim index's order, column r at r * B
    const int64_t* vpre;       // [R * B]: their inclusive prefix sums within each node's segment
    uint32_t* unres;           // [n_chunks * P]: partial unresolvable counts of the scan
};
// k_fit_preempt_scan's pods per warp, and its launch geometry (direct_grid's rule)
constexpr uint32_t FIT_PREEMPT_PODS_PER_WARP = 1;
DirectGrid fit_preempt_grid(uint32_t P, uint32_t Npad, int sms);
// the R request columns after build_victim_index: breq [B * R] (bound pod b's request of r at b * R + r) gathered
// through vx.idx into fa.vres, then scanned per segment into fa.vpre
cudaError_t build_fit_victim_index(const VictimIndex& vx, const int64_t* breq, const FitPreemptArgs& fa, uint32_t N,
                                   cudaStream_t st);
// out[P], victims[P * max_victims] (may be null) and unres[P] (may be null), device memory.  With nt.N == 0 only the rows
// and counts are written (no plan).
cudaError_t launch_fit_preempt(const NodeTable& nt, const PodView& pv, const int32_t* pod_prio, const VictimIndex& vx,
                               const FitPreemptArgs& fa, uint32_t max_victims, const PreemptPartials& part,
                               const DirectGrid& g, ks_preemption* out, int32_t* victims, uint32_t* unres,
                               cudaStream_t st);

// drain simulation (ks_drain_check).  Candidates are in the host's round order (pod count descending), so the pods of
// round r - pod r of every candidate that has one - are the first R_r candidates; slot j of every round is candidate j.
// Each candidate's moves are an overlay sorted by node, (node, f_cpu, f_mem) with f its private free, kept in
// [pod_base[j], pod_base[j] + ov_cnt[j]) of the overlay arrays.  Device memory.
struct DrainArgs {
    const int32_t* cand_node; // [D] the candidate's own node
    const uint32_t* pod_base; // [D] its first pod in the caller's order (and its overlay's base)
    const uint32_t* cand_id;  // [D] its index in the caller's order
    const uint32_t* excl;     // [Npad / 32] bits of the nodes that are no destination of any candidate, or null
    uint32_t* ov_cnt;         // [D] overlay entries, zeroed before round 0
    uint32_t* failed;         // [D] 1 once a pod of the candidate found no destination, zeroed before round 0
    int32_t* ov_node;         // [P]
    int64_t* ov_fc;           // [P]
    int64_t* ov_fm;           // [P]
    int32_t* out_idx;         // [P] caller's order, -1 before the call
    int64_t* out_score;       // [P] caller's order, 0 before the call
    uint32_t* placed;         // [D] caller's order, 0 before the call
};
// one round: the node scan for pod r of the pv.P running candidates, then their commit.  part holds g.n_chunks * pv.P
// keys and indices.
cudaError_t launch_drain_round(const NodeTable& nt, const PodView& pv, const DrainArgs& da, int policy, uint32_t r,
                               const PartialView& part, const DirectGrid& g, cudaStream_t st);

// drain simulation under the full filter (ks_fit_drain_check).  DrainArgs for the candidates and the overlay, plus what
// the scan and the commit read beyond ks_drain_check's inputs: the round's pod requests and groups, the free amounts and
// the rule words of ks_node_bind, and R more overlay columns.  With refusal words, the commit that stops a candidate
// copies its stopping pod to the candidate's slot of the stop arrays, and one counting scan over those slots follows the
// last round.  Device memory.
struct FitDrainArgs {
    uint32_t R;                // [0, KS_BIND_MAX_RESOURCES]
    uint32_t P;                // pods of the call: the stride of ov_fr's columns
    const int64_t* req;        // [P_r * R]: the round's pod j's request of r at j * R + r (the count pass: stop_req)
    const int32_t* group;      // [P_r]: the round's pods' groups, each in [-1, G) (the count pass: stop_grp)
    const int64_t* node_free;  // [R * N]
    const uint32_t* ncls;      // [G + 1]: the class of group g at g + 1, of group -1 at 0
    const uint32_t* nrules;    // [C * N], written by k_node_rules_setup
    int64_t* ov_fr;            // [R * P]: f_r of overlay entry k of candidate j at r * P + pod_base[j] + k
    int64_t *stop_cpu, *stop_mem; // [D] the stopping pod of candidate slot j; all five null without refusal words
    uint64_t* stop_sel;        // [D * W]
    int64_t* stop_req;         // [D * R]
    int32_t* stop_grp;         // [D]
    const uint32_t* stopped;   // [D] the count pass: the rounds' failed flags (its own DrainArgs::failed reads 0)
    uint32_t* refused;         // [4 * D] caller's order, zeroed before the count pass
};
// k_fit_drain_scan's pods per warp, and its launch geometry (direct_grid's rule)
constexpr uint32_t FIT_DRAIN_PODS_PER_WARP = 1;
DirectGrid fit_drain_grid(uint32_t P, uint32_t Npad, int sms);
// one round of ks_fit_drain_check: the scan for pod r of the pv.P running candidates, then their commit.  part holds
// g.n_chunks * pv.P keys and indices.
cudaError_t launch_fit_drain_round(const NodeTable& nt, const PodView& pv, const DrainArgs& da, const FitDrainArgs& fa,
                                   int policy, uint32_t r, const PartialView& part, const DirectGrid& g, cudaStream_t st);
// the refusal words after the last round: the counting scan over the D candidate slots, pv = the stop arrays
cudaError_t launch_fit_drain_refusals(const NodeTable& nt, const PodView& pv, const DrainArgs& da,
                                      const FitDrainArgs& fa, const DirectGrid& g, cudaStream_t st);

// scale-up estimate (ks_scaleup_estimate, ks_scaleup.cu).  T templates, each packed on its own by one CTA of
// k_scaleup_pack; the grid holds `slots` CTAs, CTA b takes templates b, b + slots, ... and sorts in its own scratch
// slot of 2 * pv.P entries.  Device memory.
struct ScaleupArgs {
    uint32_t T;
    const int64_t *alloc_cpu, *alloc_mem, *free_cpu, *free_mem; // [T]
    const uint64_t* labels;                                      // [T * W], row-major like the pods' selectors
    const uint32_t* max_nodes;                                   // [T]
    ks_scaleup_option* rows;                                     // [T]
    int32_t* out_node;                                           // [T * P], -1 before the call, or null
    uint32_t* reasons;                                           // [P][4] in ks_pod_reasons order, or null
    uint32_t* scratch;                                           // [slots * 2 * P]
    uint32_t slots;
};
uint32_t scaleup_slots(uint32_t T, int sms);
cudaError_t launch_scaleup(const PodView& pv, uint32_t W, const ScaleupArgs& a, cudaStream_t st);

// scale-up estimate under the full filter (ks_fit_scaleup_estimate, ks_scaleup.cu): ScaleupArgs (its `reasons` unused)
// plus ks_fit_bind's resources and rule words with the templates as the nodes.  Device memory.
struct FitScaleupArgs {
    uint32_t R;               // [0, KS_BIND_MAX_RESOURCES]
    const int64_t* req;       // [P * R]: pod p's request of r at p * R + r
    const int32_t* group;     // [P], each in [-1, G)
    const int64_t* node_free; // [R * T]: one empty node of template t, resource r at r * T + t
    const uint32_t* ncls;     // [G + 1]: the class of group g at g + 1, of group -1 at 0
    const uint32_t* nrules;   // [C * T], written by k_node_rules_setup over the templates
    int64_t* used;            // [T * R] the placed pods' requests per template, or null
    uint32_t* refused;        // [P][4] the refusal words, or null
};
// k_fit_scaleup_pack, then with f.refused k_fit_scaleup_reasons
cudaError_t launch_fit_scaleup(const PodView& pv, uint32_t W, const ScaleupArgs& a, const FitScaleupArgs& f,
                               cudaStream_t st);

// replica placement (ks_place_replicas, ks_replicas.cu).  T specs, each evaluated on its own over the node table by a
// grid of (node chunk, spec) CTAs: a scan, a fixed number of threshold-search passes, the tie split and, with the copy
// list, one CTA per spec that sorts its copies.  Device memory.
struct RepSpec;  // per-spec search state (ks_replicas.cu)
struct RepChunk; // per-(spec, node chunk) partial sums
struct ReplicaArgs {
    uint32_t T;
    const int64_t *req_cpu, *req_mem; // [T]
    const uint64_t* sel;              // [T * W], row-major
    const uint32_t* replicas;         // [T]
    const uint64_t* offset;           // [T]: first copy of spec t in the copy list
    ks_replica_plan* rows;            // [T]
    int32_t* out_node;                // [sum of replicas], -1 before the call, or null (no copy list)
    int64_t* out_score;               // [sum of replicas], 0 before the call; set exactly when out_node is
    RepSpec* spec;                    // [T]
    RepChunk* chunk;                  // [T * n_chunks]
    int32_t* copy_node;               // [sum of replicas] copies in node-then-copy order, with out_node
    int64_t* copy_score;
    uint32_t* sort_buf;               // [2 * sum of replicas], with out_node
    uint32_t n_chunks, chunk_len;     // node chunks per spec and nodes per chunk (a multiple of 256)
};
// KS_SCORE_LEAST_BALANCED places the copies one at a time (k_rep_seq): per CTA, device scratch for every node
struct ReplicaSeqArgs {
    int64_t* score;        // [ctas * N] current score of every node, INT64_MIN when it takes no further copy
    uint32_t* placed;      // [ctas * N] copies placed on every node
    uint32_t ctas, block;  // the grid, and nodes per block maximum
};
size_t replica_spec_bytes(uint32_t T);
size_t replica_chunk_bytes(uint32_t T, uint32_t n_chunks);
void replica_chunks(uint32_t N, uint32_t T, int sms, uint32_t* n_chunks, uint32_t* chunk_len);
// KS_SCORE_LEAST_BALANCED's sequential placement: its CTAs (12 bytes of scratch per node each, 64 MiB in all or one
// CTA's worth) and the nodes per block maximum
void replica_seq_grid(uint32_t N, uint32_t T, int sms, uint32_t* ctas, uint32_t* block);
cudaError_t launch_replicas(const NodeTable& nt, int policy, const ReplicaArgs& a, const ReplicaSeqArgs& q,
                            cudaStream_t st);

// topology spread for replica placement (ks_place_replicas_spread and _multi, ks_spread.cu).  The specs come as
// ReplicaArgs' T, requests, selectors, replicas, offsets and copy list (its rows and search state are not used).  Device
// memory.  Internal key 0 is the primary, the key with the fewest domains; keys 1 .. K-1 are the secondaries.
struct SpreadOrder {              // k_spread_order's input and outputs for one key, once per call
    const int32_t* node_domain;   // [N]
    uint32_t* sort_buf;           // [2N]
    uint32_t* perm;               // [N]: nodes with a domain by (domain, node), the rest after dstart[D]
    uint32_t* pos;                // [N]: node -> position in perm
    uint32_t* dstart;             // [D + 1]: domain d's nodes are perm[dstart[d] .. dstart[d + 1])
    uint32_t D;
};
struct SpreadOrders {             // one k_spread_order CTA per key
    SpreadOrder key[KS_SPREAD_MAX_KEYS];
    uint32_t K;
};
struct SpreadArgs {
    uint32_t D;                   // the primary's
    const int32_t* node_domain;   // [N]
    const uint32_t *perm, *pos, *dstart;
    const uint32_t* max_skew;     // [T * K]
    const uint32_t* min_domains;  // [T * K] or null
    const uint32_t* existing;     // [T * S] or null
    ks_spread_plan* rows;         // [T * K]
    uint32_t* out_count;          // [T * S] or null
    unsigned char* scratch;       // [bytes of spread_seq_grid]
    uint32_t ctas;
};
// K >= 2 only (the single-key kernel reads none of it, and takes it as a separate parameter so that its own code stays
// as it was): per internal key i, its column col[i] in the caller's key order (max_skew, min_domains and rows are strided
// by K), its count offset off[i] = P_col[i] (existing and out_count are strided by S = sum of D_k), its domains Dk[i]
// and its order (dom[0] = SpreadArgs::node_domain)
struct SpreadKeys {
    uint32_t K, S;
    uint32_t col[KS_SPREAD_MAX_KEYS], off[KS_SPREAD_MAX_KEYS], Dk[KS_SPREAD_MAX_KEYS];
    const int32_t* dom[KS_SPREAD_MAX_KEYS];
    const uint32_t* kperm[KS_SPREAD_MAX_KEYS];
    const uint32_t* kdstart[KS_SPREAD_MAX_KEYS];
    uint64_t cta_bytes;           // scratch per CTA
};
// k_spread_seq's scratch per CTA for the keys' domain counts Dk[0 .. K-1] (Dk[0] the primary's): 12 per node, 20 per
// primary domain and 12 per block slot, and with K >= 2 also 4 per block slot and 8 per secondary domain
uint64_t spread_cta_bytes_keys(uint32_t N, const uint32_t* Dk, uint32_t K);
// k_spread_seq's CTAs - as many as fit in 64 MiB (at least one, at most one per spec and two per SM) - and the bytes of
// their scratch
void spread_seq_grid(uint64_t cta_bytes, uint32_t T, int sms, uint32_t* ctas, uint64_t* bytes);
cudaError_t launch_spread(const NodeTable& nt, int policy, const ReplicaArgs& a, const SpreadOrders& o,
                          const SpreadArgs& q, const SpreadKeys& mk, cudaStream_t st);

} // namespace ks

namespace ks {
cudaError_t launch_stream_resolve(int64_t* free_cpu, int64_t* free_mem, const int32_t* claim_node, const int64_t* req_cpu,
                                  const int64_t* req_mem, uint32_t n, uint32_t N, uint8_t* accepted, cudaStream_t st);
uint32_t stream_max_claims();

// device-side micro-batch loop (k_stream_batch, ks_stream.cu)
constexpr uint32_t STREAM_BATCH_MAX = 1024; // pods per cooperative launch
struct StreamBatchArgs {
    uint32_t N, Npad;
    const int64_t *alloc_cpu, *alloc_mem;
    const uint64_t* labels;
    int64_t *free_cpu, *free_mem;
    int policy;
    uint32_t m;
    const int64_t *req_cpu, *req_mem;
    const uint64_t* sel;
    int64_t* pkey;  // [STREAM_BATCH_MAX * grid]
    int32_t* pidx;  // [STREAM_BATCH_MAX * grid]
    uint32_t* pend; // [2 * STREAM_BATCH_MAX]
    uint32_t* ctl;  // [2]: pending count, rounds
    int32_t* out_idx;
    int64_t* out_score;
    uint32_t max_rounds;
    uint32_t grid;
};
cudaError_t launch_stream_batch(const StreamBatchArgs& a, uint32_t W, cudaStream_t st);
// pod groups (k_gang_batch, ks_stream.cu): a.m = all pods, a.max_rounds unused (each group runs up to size + 1 rounds)
struct GangArgs {
    uint32_t n;                 // groups
    const uint32_t* offset;     // [n+1]: group g = pods [offset[g], offset[g+1]), 1..STREAM_BATCH_MAX of them
    const uint32_t* min_member; // [n]
    uint32_t* ctl;              // [2n]: per group pending count, rounds
    uint32_t* placed;           // [n]: pods the round loop bound (before any rollback)
};
cudaError_t launch_gang_batch(const StreamBatchArgs& a, const GangArgs& g, uint32_t W, cudaStream_t st);

// The bind calls (ks_spread_bind.cu), one mode each: ks_spread_bind, ks_affinity_bind, ks_profile_bind, ks_node_bind
// with rules, ks_fit_bind and ks_gang_fit_bind.  Each mode filters as the one before it and adds rules; PROFILE and NODE
// also add scores; FIT is NODE with the scalar resources after fit and selector; GANG_FIT is FIT with the pods cut into
// gangs that commit or roll back whole.
enum BindMode { BIND_SPREAD, BIND_AFFINITY, BIND_PROFILE, BIND_NODE, BIND_FIT, BIND_GANG_FIT };
// Refusal words and score parts per pod in a mode's outputs (include/ksched.h)
__host__ __device__ constexpr uint32_t bind_refusal_words(BindMode m) {
    return m == BIND_FIT || m == BIND_GANG_FIT ? 5 : m == BIND_NODE ? 4 : m == BIND_SPREAD ? 1 : 2;
}
__host__ __device__ constexpr uint32_t bind_part_words(BindMode m) {
    return m == BIND_NODE || m == BIND_FIT || m == BIND_GANG_FIT ? 5 : 3;
}

// topology spread when binding (ks_spread_bind), the state of every mode.  Device memory.  Key k's domains are the
// counts [Pk[k], Pk[k] + Dk[k]) of each group's S.
struct SpreadBindArgs {
    uint32_t N, Npad, P, G, K, S;
    uint32_t Dk[KS_SPREAD_MAX_KEYS], Pk[KS_SPREAD_MAX_KEYS];
    const int64_t *alloc_cpu, *alloc_mem;
    const uint64_t* labels;
    int64_t *free_cpu, *free_mem;   // charged
    int policy;
    const int64_t *req_cpu, *req_mem; // [P]
    const uint64_t* sel;              // [P * W], row-major
    const int32_t* group;             // [P], each in [-1, G)
    const uint64_t* gsel;             // [G * W]: each group's selector (the same in all its pods)
    const int32_t* dom;               // [K * N]: key k's node_domain at k * N
    const uint32_t* max_skew;         // [G * K], 0 = key not constrained
    const uint32_t* min_domains;      // [G * K] or null
    const uint32_t* existing;         // [G * S] or null
    uint8_t* elig;                    // [G * S] eligible-domain flags
    uint32_t* gk;                     // [G * K * 4] per (group, key): m, domains at m, |E|, flags
    uint32_t* cnt;                    // [G * S] counts, final after the call
    int64_t* pkey;                    // [grid] per-CTA partials
    int32_t* pidx;
    uint32_t* pref;
    int32_t* out_idx;                 // [P]
    int64_t* out_score;               // [P]
    uint32_t* out_refused;            // [bind_refusal_words(mode) * P]
    uint32_t grid, setup_grid;        // the walk's CTAs; k_bind_setup's, one per group, grid-strided
    // inter-pod affinity (read by every mode but SPREAD).  Counter arrays B_{g,k} / A_{g,k} of D_k words
    // in acnt; one word per group at acnt[any_base + g] is set once a pod of M_g is bound on a node that carries one of
    // g's affinity keys.  Update entry: h | k << 16 | kind << 20 (kind 0 = B, 1 = A) raises that array of group h.
    const uint32_t* abase;            // [G * K * 2]: base of B_{g,k}, then of A_{g,k}, in acnt; AFF_NONE = no array
    const uint32_t* aflag;            // [G]: AFF_SELF when g is in M_g
    const uint32_t* upd_off;          // [G + 1]: group h's update entries
    const uint32_t* upd;
    const int32_t *ex_group, *ex_node; // [E] existing pods
    uint32_t E, any_base, aff_grid;
    uint32_t* acnt;                   // counters, zeroed by the launcher
    uint32_t* paref;                  // [grid] per-CTA affinity refusals
};
uint32_t bind_setup_grid(uint32_t G, int sms);
constexpr uint32_t AFF_NONE = 0xffffffffu, AFF_SELF = 1u;

// Every bind kernel takes this: ks_affinity_bind's state in b, first, so that its fields keep their parameter offsets,
// then the soft terms of ks_profile_bind (DESIGN.md 5o) and the node rules of ks_node_bind.  The soft counts scnt start
// at existing (or 0), the IPA counters I_{g,k} (int64, D_k words each at ibase[g * K + k] in icnt) at 0 before the
// existing pods' entries.  Update entry of group h: g | k << 16 with coefficient icoef, added to I_{g,k}[d_k(n)] when a
// pod of h binds on n.  Per node of the slice, pass 1 leaves iraw[n] = its IPA raw, or PB_NOT_CAND when n is not a
// candidate, and pass 2 praw[n] = its PodTopologySpread raw, or -1 when it is ignored.
constexpr uint32_t PB_SH_WORDS = 64; // domains below 64 * 32 of each key are marked in a per-CTA bitmap first
struct ProfileBindArgs {
    SpreadBindArgs b;
    const uint32_t* soft_skew;        // [G * K], 0 = no soft constraint on the key
    const uint8_t* soft_all;          // [G]
    const double* logw;               // [N + 2]: log(size + 2)
    uint32_t uniq;                    // bit k: key k has at most one node per domain (size_k counts nodes)
    uint32_t bwo[KS_SPREAD_MAX_KEYS]; // word offset of key k in each parity's domain bitmap
    uint32_t BW;                      // words per parity
    uint32_t* bits;                   // [2 * BW], zeroed by the launcher; pod p marks parity p & 1
    uint32_t* scnt;                   // [G * S] soft counts, final after the call
    const uint32_t* ibase;            // [G * K], AFF_NONE = no IPA counters
    const uint32_t* iupd_off;         // [G + 1]
    const uint32_t* iupd;
    const int32_t* icoef;
    int64_t* icnt;                    // IPA counters, zeroed by the launcher
    uint64_t iwords;
    int64_t *iraw, *praw;             // [N]
    uint32_t* pdom;                   // [grid * KS_SPREAD_MAX_KEYS] per-CTA partials: new domains per soft key
    uint32_t* plack;                  // [grid]: soft keys some non-ignored candidate lacks
    int64_t *pimin, *pimax, *ppmin, *ppmax; // [grid]: IPA raw and PodTopologySpread raw extremes
    int64_t* out_parts;               // [bind_part_words(mode) * P]
    uint32_t wspread, waff;
    // ks_node_bind (DESIGN.md 5p; read by NODE only).  Rule word of (class c, node n) at nrules[c * N + n]:
    // NR_REASON bits (0 pass, NR_TAINT, NR_AFFINITY), NR_AFF_OK, the PreferNoSchedule count at NR_TT_SHIFT and the
    // preferred NodeAffinity raw at NR_NA_SHIFT.  Class c's terms [cterm_off[c], cterm_off[c + 1]): weight cterm_w (0 =
    // required), expressions [cexpr_off[t], cexpr_off[t + 1]): key cexpr_key, set at word cexpr_set of nset.
    const uint32_t* ncls;             // [G + 1]: the class of group g at g + 1, of group -1 at 0
    uint32_t* nrules;                 // [C * N], written by k_node_rules_setup
    uint32_t C, KN, NDk[KS_NODE_RULES_MAX_KEYS];
    const int32_t* ndom;              // [KN * N]
    const uint64_t *taint_hard, *taint_soft; // [N]
    const uint64_t* ctol;             // [2C]: hard, soft tolerations
    const uint32_t *cterm_off, *cterm_w, *cexpr_off, *cexpr_key;
    const uint64_t *cexpr_set, *nset;
    uint32_t *ptref, *pnref;          // [grid] per-CTA taint and node-affinity refusals
    uint32_t *ptmax, *pnmax;          // [grid] per-CTA maxima of the two raws over the candidates
    uint32_t wtaint, wnaff, rules_grid;
    // ks_fit_bind (DESIGN.md 5r; read by FIT only), after every other field so that theirs keep their parameter
    // offsets.  Resource r of node n at r * N + n, laid out like free_cpu; pod p's request of r at p * R + r.
    uint32_t R;                       // [0, KS_BIND_MAX_RESOURCES]
    const int64_t* res_req;           // [P * R], each >= 0
    const int64_t* res_node_free;     // [R * N]: the caller's node_free, copied into res_free by the launcher
    int64_t* res_free;                // [R * N]: charged, final after the call
    uint32_t* pfref;                  // [grid] per-CTA resource refusals
    // ks_gang_fit_bind (DESIGN.md 5s; read by GANG_FIT only), after every other field.  Gang j is the pods
    // [goff[j], goff[j + 1]); after its last pod it commits when at least gmin[j] of them bound, else rolls back.  The
    // rollback lists, once each, the groups whose gk words and the groups whose any-flag it recomputes: gmark[g] and
    // gmark[G + h] hold the last gang (j + 1) that listed them, glist the lists.
    uint32_t n_gangs;
    const uint32_t* goff;             // [n_gangs + 1]
    const uint32_t* gmin;             // [n_gangs]
    uint32_t* gplaced;                // [n_gangs]: the pods of the gang that bound, before any rollback
    uint32_t* gmark;                  // [2G], zeroed by the launcher
    uint32_t* glist;                  // [2G]
};
constexpr int64_t PB_NOT_CAND = INT64_MIN;
constexpr uint32_t NR_REASON = 3u, NR_TAINT = 1u, NR_AFFINITY = 2u, NR_AFF_OK = 4u, NR_TT_SHIFT = 3, NR_NA_SHIFT = 10;
// One bind call's launches, in order: (NODE, FIT) k_node_rules_setup; k_bind_setup when G > 0; (every mode but SPREAD)
// the counters zeroed, (PROFILE, NODE, FIT) the IPA counters and the bitmaps zeroed and the soft counts set, (FIT)
// res_free set from res_node_free, (GANG_FIT) gmark zeroed, then k_affinity_setup and (PROFILE, NODE, FIT)
// k_profile_setup over the existing pods when E > 0; then the walk k_bind_seq, one cooperative launch of grid CTAs.  FIT
// includes GANG_FIT here.  The fields a mode does not read may be left zero.
cudaError_t launch_bind(BindMode mode, const ProfileBindArgs& a, uint64_t acnt_words, uint32_t W, cudaStream_t st);
// k_node_rules_setup alone: the rule words nrules [C * N] from the NODE fields of a and a.b.N (launch_bind's first
// launch in NODE and FIT; ks_fit_preempt's rule words)
cudaError_t launch_node_rules(const ProfileBindArgs& a, cudaStream_t st);
} // namespace ks
